"""INTEGRATION.md binding B1 measured: `b200_upfirdn2d_f32` in the reference's own tensor convention ([N*C, H, W, 1],
op/upfirdn2d.py:99) against the reference's JIT-compiled `upfirdn2d_op` (op/upfirdn2d_kernel.cu, from oracle/_ref,
unmodified) on the same GPU tensors, for the three parameterisations NCSN++ uses.  Prints one markdown table:

    python tools/bench_upfirdn2d.py [--md OUT.md]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench                                                # noqa: E402
from score_sde_pytorch_b200.op import upfirdn2d as ours_upfirdn2d     # noqa: E402  (the function; the package re-exports it)

ap = argparse.ArgumentParser()
ap.add_argument('--md', default=None)
ap.add_argument('--reps', type=int, default=20)
args = ap.parse_args()
dev = torch.device('cuda:0')
try:
  bench.import_reference()
  from op import upfirdn2d as ref_upfirdn2d                # the reference's Python wrapper over its pybind module
except Exception as e:                                      # noqa: BLE001
  ref_upfirdn2d = None
  print('reference op unavailable:', e)

k = np.outer([1, 3, 3, 1], [1, 3, 3, 1]).astype(np.float32)
k /= k.sum()
cases = [('downsample_2d (down=2, pad 1,1)', (1024, 128, 32, 32), k, 1, 2, (1, 1)),
         ('upsample_2d (up=2, pad 2,1, gain 4)', (1024, 256, 16, 16), k * 4, 2, 1, (2, 1)),
         ('pyramid pad (pad 2,2)', (1024, 3, 32, 32), k, 1, 1, (2, 2)),
         ('downsample_2d 256x256 planes', (64, 128, 256, 256), k, 1, 2, (1, 1))]


def timed(fn):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(args.reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / args.reps


lines = ['# upfirdn2d in the reference layout [N*C, H, W, 1]: this library vs the reference\'s own JIT kernel (binding B1)',
         '| case | tensor | ours ms | GB/s | reference ms | GB/s | speed-up | max abs diff |', '|---|---|---:|---:|---:|---:|---:|---:|']
for name, shape, kk, up, down, pad in cases:
  torch.manual_seed(0)
  x = torch.randn(*shape, device=dev)
  kt = torch.tensor(kk, device=dev)
  y = ours_upfirdn2d(x, kt, up=up, down=down, pad=pad)
  nbytes = (x.numel() + y.numel()) * 4
  t_ours = timed(lambda: ours_upfirdn2d(x, kt, up=up, down=down, pad=pad))
  if ref_upfirdn2d is not None:
    yr = ref_upfirdn2d(x, kt, up=up, down=down, pad=pad)
    t_ref = timed(lambda: ref_upfirdn2d(x, kt, up=up, down=down, pad=pad))
    diff = float((y - yr).abs().max())
    lines.append(f'| {name} | {list(shape)} | {t_ours:.3f} | {nbytes / t_ours / 1e6:.0f} | {t_ref:.3f} | {nbytes / t_ref / 1e6:.0f} | {t_ref / t_ours:.2f}x | {diff:.1e} |')
  else:
    lines.append(f'| {name} | {list(shape)} | {t_ours:.3f} | {nbytes / t_ours / 1e6:.0f} | n/a | | | |')
txt = '\n'.join(lines)
print(txt)
if args.md:
  with open(args.md, 'w') as f:
    f.write(txt + '\n(timings include each side\'s Python wrapper: output allocation and, on our side, the 16-tap host array)\n')
