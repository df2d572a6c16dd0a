"""Launch plans of the engine for a fixed matrix of configurations, as JSON: the parameter table, the weight and workspace
sizes, every op of the bound plan in order (label, kind, flops, algorithmic bytes), the launches per forward and, for a
few PC samplers, the launches per step and the PC workspace size.

  python tools/dump_engine_plans.py --out tests/golden/engine_plans.json.gz   (binding a plan needs a GPU)

tests/test_gpu_engine_plans.py rebuilds the matrix on a GPU and requires the plans to equal the golden exactly;
tests/test_engine_plans_cpu.py checks the parts that are planned without a device (parameter tables, weight and
workspace sizes).  The matrix reaches every op the plan builder can emit: each precision, the lane split, both halo
forms, both heads, the tangent plans, the few-channel levels with GroupNorm on load (tf32) and behind a separate
GroupNorm pass (tf32x3), and the input_skip / output_skip pyramids of the high-resolution networks."""
import argparse
import ctypes
import gzip
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (REPO, os.path.join(REPO, 'tests')):
  if _p not in sys.path:
    sys.path.insert(0, _p)

from helpers import golden_config                  # noqa: E402
from score_sde_pytorch_b200 import _lib, configs   # noqa: E402

GOLDEN = os.path.join(REPO, 'tests', 'golden', 'engine_plans.json.gz')
WS_BATCHES = (1, 8, 256)   # workspace sizes are recorded at these batches and at the case's own


def _config(name):
  if name == 'nf16_progressive':
    # the nf = 16 few-channel network of test_few_channel_levels_groupnorm_on_load_matches_oracle
    return configs.tiny_progressive(nf=16, image_size=64, num_res_blocks=2, ch_mult=(1, 2, 2, 4), attn_resolutions=(8,))
  if name == 'tiny_ddpm':
    return configs.tiny_ddpm()
  if name == 'vp_cifar10_ddpm_continuous':
    return configs.vp_cifar10_ddpm_continuous()
  return golden_config(name)


def _case(name, precision, batch=8, tangent=False, pc=(), **options):
  key = '/'.join([name, precision, f'b{batch}'] + (['tangent'] if tangent else []) +
                 [f'{k}={v}' for k, v in sorted(options.items())])
  return dict(key=key, name=name, precision=precision, batch=batch, tangent=tangent, pc=tuple(pc), options=options)


def cases():
  out = [_case('cifar10_ve', p, pc=('ve_rd_langevin',) if p == 'f16' else ()) for p in ('f16', 'tf32', 'fp32')]
  out += [_case('cifar10_ve', 'f16', batch=256, lanes=2), _case('cifar10_ve', 'f16', halo=False),
          _case('cifar10_ve', 'tf32', cuda_core_head=True)]
  for name, precisions in (('cifar10_ddpmpp', ('tf32',)), ('vp_cifar10_ddpm_continuous', ('f16', 'tf32'))):
    out += [_case(name, p) for p in precisions]
    out += [_case(name, p, tangent=True) for p in ('tf32', 'fp32')]
  pcs = {'tiny': ('ve_rd_langevin', 've_ald', 'inpaint', 'colorize'), 'tiny_vp': ('vp_em',)}
  for name in ('tiny', 'tiny_vp', 'tiny_noattn', 'tiny_progressive', 'tiny_ddpm', 'tiny_ddpmpp'):
    out += [_case(name, p, pc=pcs.get(name, ()) if p == 'tf32' else ()) for p in ('fp32', 'tf32')]
    if name in ('tiny_ddpm', 'tiny_ddpmpp'):
      out += [_case(name, p, tangent=True) for p in ('fp32', 'tf32')]
  out.append(_case('tiny', 'tf32', keep_activations=True))
  out += [_case('nf16_progressive', p) for p in ('tf32', 'tf32x3')]
  out += [_case(name, 'tf32', batch=1) for name in ('celebahq_256', 'ffhq_1024')]
  return out


def make_model(case):
  """The engine-backed module of a case, with deterministic weights."""
  from score_sde_pytorch_b200.models.ddpm import DDPM
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  cfg = _config(case['name'])
  torch.manual_seed(0)
  cls = DDPM if cfg.model.name == 'ddpm' else NCSNpp
  return cls(cfg, precision=case['precision'], **case['options'])


def _native_config(model, tangent):
  c = model._native_config()
  c.tangent = int(tangent)
  return c


def planned_record(case, model=None):
  """What the engine plans without a device: parameter table, weight blob size, workspace size at each batch."""
  model = model or make_model(case)
  lib = _lib.load()
  h = ctypes.c_void_p()
  _lib.call('b200_ncsnpp_create', ctypes.byref(_native_config(model, case['tangent'])), ctypes.byref(h))
  try:
    params = [[name, list(shape)] for name, shape in model._param_table(h)]
    ws = {str(b): int(lib.b200_ncsnpp_workspace_bytes(h, b)) for b in sorted(set(WS_BATCHES) | {case['batch']})}
    return dict(params=params, weights_bytes=int(lib.b200_ncsnpp_weights_bytes(h)), workspace_bytes=ws)
  finally:
    lib.b200_ncsnpp_destroy(h)


def _pc_record(model, kind, batch, device):
  from score_sde_pytorch_b200 import native, sde_lib
  R, C = model.config.data.image_size, model.config.data.num_channels
  shape = (batch, C, R, R)
  ve, vp = sde_lib.VESDE(0.01, 50, 10), sde_lib.VPSDE(0.1, 20., 10)
  if kind == 'vp_em':
    plan = native.PcPlan(model, vp, 'euler_maruyama', 'none', shape, 0.16, 1, False, 1e-3, device)
  elif kind == 've_ald':
    plan = native.PcPlan(model, ve, 'none', 'ald', shape, 0.16, 2, False, 1e-5, device)
  elif kind in ('inpaint', 'colorize'):
    plan = native.ConstrainedPcPlan(model, ve, 'reverse_diffusion', 'langevin', shape, 0.16, 1, False, 1e-5, device, kind)
  else:
    plan = native.PcPlan(model, ve, 'reverse_diffusion', 'langevin', shape, 0.16, 1, False, 1e-5, device)
  plan._ensure()
  lib = _lib.load()
  rec = dict(launches_per_step=int(lib.b200_pc_launches_per_step(plan._pc)),
             workspace_bytes=int(lib.b200_pc_workspace_bytes(plan._pc)))
  plan._release()
  return rec


def bound_record(case, device):
  """The full record of a case: the planned part plus the op table of the plan bound on `device`."""
  model = make_model(case).to(device)
  rec = planned_record(case, model)
  eng = model.engine(case['batch'], device, tangent=case['tangent'])
  lib, h = _lib.load(), eng['h']
  name, kind, flops, nbytes = ctypes.create_string_buffer(256), ctypes.c_int(), ctypes.c_double(), ctypes.c_double()
  ops = []
  for i in range(int(lib.b200_ncsnpp_num_ops(h))):
    _lib.call('b200_ncsnpp_op_info', h, i, name, 256, ctypes.byref(kind), ctypes.byref(flops))
    _lib.call('b200_ncsnpp_op_bytes', h, i, ctypes.byref(nbytes))
    ops.append([name.value.decode(), kind.value, flops.value, nbytes.value])
  rec['ops'] = ops
  rec['launches_per_forward'] = int(lib.b200_ncsnpp_launches_per_forward(h))
  rec['pc'] = {k: _pc_record(model, k, case['batch'], device) for k in case['pc']}
  model._release()
  return rec


def dump(device):
  return {c['key']: bound_record(c, device) for c in cases()}


def write(plans, path):
  """gzip-compressed JSON (header without a timestamp, so the same plans give the same bytes)."""
  with open(path, 'wb') as raw, gzip.GzipFile(filename='', fileobj=raw, mode='wb', mtime=0) as fh:
    fh.write(json.dumps(plans, indent=1).encode())


def load(path=GOLDEN):
  with gzip.open(path, 'rt') as fh:
    return json.load(fh)


if __name__ == '__main__':
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', required=True)
  args = ap.parse_args()
  plans = dump(torch.device('cuda:0'))
  write(plans, args.out)
  print(f'{len(plans)} plans, {sum(len(r["ops"]) for r in plans.values())} ops -> {args.out}')
