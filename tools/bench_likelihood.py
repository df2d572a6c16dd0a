#!/usr/bin/env python
"""Bits/dim on the engine: DDPM cont. CIFAR-10 (``configs/vp/ddpm/cifar10_continuous.py``), VP SDE, the reference's
``get_likelihood_fn`` defaults (Rademacher, RK45, rtol = atol = 1e-5, eps = 1e-5), batch 128.

The data are seeded, uniformly dequantised random 8-bit "images" (no dataset is read), scaled to [-1, 1] like the
config's centred data.  Weights are the random init with the zero-initialised weights re-drawn at scale 1,
``torch.manual_seed(0)``.  Reported: NFE and wall time of one full likelihood computation through
``score_sde_pytorch_b200.likelihood`` (device-resident solve, one primal+tangent evaluation per right-hand side); the
CUDA-event time of one primal+tangent evaluation (``model.jvp``) against one primal forward; and, as the baseline, the
same batch through the reference's own ``likelihood_fn`` and DDPM on the GPU (the unmodified copy under oracle/_ref,
autograd VJP divergence, scipy host loop).  The GPU's name and power limit are read in the same run.

    python tools/bench_likelihood.py [--precision tf32] [--skip-reference]

One JSON line on stdout.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench import ClockSampler, import_reference   # noqa: E402
from bench_ddpm import gpu_identity   # noqa: E402


def event_ms(fn, warmup=3, iters=10):
  for _ in range(warmup):
    fn()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=128)
  ap.add_argument('--precision', default='tf32', choices=['tf32', 'fp32'])
  ap.add_argument('--skip-reference', action='store_true')
  args = ap.parse_args()

  from oracle import ddpm_oracle
  from score_sde_pytorch_b200 import configs, likelihood, sde_lib
  from score_sde_pytorch_b200.models.ddpm import DDPM
  dev = torch.device('cuda:0')
  cfg = configs.vp_cifar10_ddpm_continuous()
  torch.manual_seed(0)
  model = DDPM(cfg, precision=args.precision)
  sd = ddpm_oracle.redraw_zero_init(model.state_dict())
  model.load_state_dict(sd)
  model = model.to(dev)
  sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales)
  g = torch.Generator().manual_seed(3)
  B = args.batch
  data = ((torch.randint(0, 256, (B, 3, 32, 32), generator=g).float() + torch.rand(B, 3, 32, 32, generator=g)) / 256.)
  data = (data * 2. - 1.).to(dev)
  inverse_scaler = lambda x: (x + 1.) / 2.
  name, power = gpu_identity(0)

  labels = torch.full((B,), 500.0, device=dev)
  v = torch.randint_like(data, 0, 2) * 2 - 1.
  with torch.no_grad():
    ms_fwd = event_ms(lambda: model(data, labels, labels_uniform=True))
    ms_jvp = event_ms(lambda: model.jvp(data, labels, v, labels_uniform=True))

  fn = likelihood.get_likelihood_fn(sde, inverse_scaler)
  clocks = ClockSampler(0)
  clocks.start()
  torch.cuda.manual_seed(7)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  bpd, z, nfe = fn(model, data)
  torch.cuda.synchronize()
  wall = time.perf_counter() - t0
  clk = clocks.stop()

  ref = dict(wall_s='not measured', nfe='not measured', bpd_mean='not measured')
  if not args.skip_reference:
    try:
      ns = import_reference()
      import importlib
      importlib.import_module('models.ddpm')
      ref_lik = importlib.import_module('likelihood')
      ref_sde = ns.sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales)
      rcfg = configs.vp_cifar10_ddpm_continuous()
      rcfg.device = dev
      rmodel = ns.mutils.get_model('ddpm')(rcfg).to(dev).eval()
      rmodel.load_state_dict({k: t.to(dev) for k, t in sd.items()}, strict=True)
      rfn = ref_lik.get_likelihood_fn(ref_sde, inverse_scaler)
      torch.cuda.manual_seed(7)
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      rbpd, _, rnfe = rfn(rmodel, data)
      torch.cuda.synchronize()
      ref = dict(wall_s=round(time.perf_counter() - t0, 3), nfe=int(rnfe), bpd_mean=round(float(rbpd.mean()), 6))
    except (ImportError, FileNotFoundError, RuntimeError) as e:
      ref['error'] = f'{type(e).__name__}: {e}'[:300]

  print(json.dumps(dict(
      metric='bits/dim wall time, DDPM cont. CIFAR-10 VP, RK45 rtol=atol=1e-5, Rademacher, batch %d' % B,
      value=round(wall, 3), unit='s', higher_is_better=False,
      gpu=name, power_limit_w=power, batch=B, precision=args.precision, nfe=int(nfe),
      bpd_mean=round(float(bpd.mean()), 6), finite=bool(torch.isfinite(bpd).all() and torch.isfinite(z).all()),
      solver=fn.last_stats.get('solver'), ms_per_forward=round(ms_fwd, 4), ms_per_jvp=round(ms_jvp, 4),
      jvp_over_forward=round(ms_jvp / ms_fwd, 3), launches_per_jvp=len(model.op_names(tangent=True)),
      launches_per_forward=model.launches_per_forward(), clocks=clk,
      reference=dict(ref, what="reference likelihood_fn + DDPM (oracle/_ref, unmodified), autograd VJP, scipy host loop, "
                              "same data, same CUDA seed"),
      config=dict(workload='configs/vp/ddpm/cifar10_continuous.py network (35.2 M parameters), 32x32',
                  weights='random init, zero-init weights re-drawn at scale 1, torch.manual_seed(0)',
                  data='uniformly dequantised random 8-bit images, torch.Generator seed 3, scaled to [-1, 1]'))))


if __name__ == '__main__':
  main()
