"""Per-op device time of one network evaluation (CUDA events around every launch, run serially on one
stream), grouped by shape label:  python tools/profile_ops.py --batch 1024 [--md OUT.md]"""
import argparse
import collections
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import headline_config                                    # noqa: E402
from score_sde_pytorch_b200 import _lib                              # noqa: E402
from score_sde_pytorch_b200.models.ncsnpp import NCSNpp              # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=1024)
ap.add_argument('--precision', default='f16')
ap.add_argument('--reps', type=int, default=5)
ap.add_argument('--md', default=None)
ap.add_argument('--config', default='headline', choices=['headline', 'celebahq_256', 'ddpmpp_256', 'ffhq_1024', 'cifar10_ddpmpp'])
ap.add_argument('--no-halo', action='store_true', help='3x3 mainloop with one shifted tile load per filter tap everywhere')
args = ap.parse_args()
dev = torch.device('cuda:0')
torch.manual_seed(0)
from score_sde_pytorch_b200 import configs                          # noqa: E402
cfg = {'headline': headline_config, 'celebahq_256': configs.ve_celebahq_256_ncsnpp_continuous,
       'ddpmpp_256': configs.subvp_celebahq_256_ddpmpp_continuous, 'ffhq_1024': configs.ve_ffhq_1024_ncsnpp_continuous,
       'cifar10_ddpmpp': configs.vp_cifar10_ddpmpp_continuous}[args.config]()
cfg.model.init_scale = 1.0
model = NCSNpp(cfg, precision=args.precision, halo=not args.no_halo).to(dev)
B = args.batch
eng = model.engine(B, dev)
h = eng['h']
n = int(_lib.load().b200_ncsnpp_num_ops(h))
R = cfg.data.image_size
x = torch.randn(B, 3, R, R, device=dev) * 10
lab = torch.full((B,), 1.0, device=dev)
out = torch.empty_like(x)
ms = (ctypes.c_float * n)()
acc = [0.0] * n
for r in range(args.reps + 2):
  _lib.call('b200_ncsnpp_profile_ops', h, _lib.ptr(x), _lib.ptr(lab), 1, _lib.ptr(out), _lib.stream_ptr(dev), ms, n)
  if r >= 2:
    for i in range(n):
      acc[i] += ms[i] / args.reps
groups = collections.OrderedDict()
name = ctypes.create_string_buffer(200); kind = ctypes.c_int(); fl = ctypes.c_double()
for i in range(n):
  _lib.call('b200_ncsnpp_op_info', h, i, name, 200, ctypes.byref(kind), ctypes.byref(fl))
  g = groups.setdefault(name.value.decode(), [0, 0.0, 0.0])
  g[0] += 1; g[1] += acc[i]; g[2] += fl.value
total = sum(acc)
lines = [f'# per-op profile ({args.config}), one network evaluation, batch {B}, {args.precision}: {n} ops, {total:.3f} ms (serial, event-timed)',
         '| op | launches | total ms | share | us/launch | TFLOP/s |', '|---|---:|---:|---:|---:|---:|']
for k, (c, t, f) in sorted(groups.items(), key=lambda kv: -kv[1][1]):
  tf = f / (t * 1e-3) / 1e12 if t > 0 and f > 0 else 0.0
  lines.append(f'| `{k}` | {c} | {t:.3f} | {100 * t / total:.1f}% | {1e3 * t / c:.1f} | {tf:.0f} |' if tf else
               f'| `{k}` | {c} | {t:.3f} | {100 * t / total:.1f}% | {1e3 * t / c:.1f} | |')
txt = '\n'.join(lines)
print(txt)
if args.md:
  with open(args.md, 'w') as fobj:
    fobj.write(txt + '\n')
