#!/usr/bin/env python
"""Multistep DPM-Solver++ sampling (``sampling.get_dpm_solver_sampler``, native loop) on NCSN++ cont. CIFAR-10 (VE,
``configs/ve/cifar10_ncsnpp_continuous.py``) and DDPM++ cont. CIFAR-10 (VP, ``configs/vp/cifar10_ddpmpp_continuous.py``)
at batch 1024 in ``'f16'``, with 10 / 20 / 50 steps at orders 2 and 3 (log-SNR grid, eps = 1e-3, no denoising step).

For each network the same process times the network forward alone (``--forwards`` uniform-label forwards between two
synchronises), then each sampler configuration (one warm-up call, which captures the step's CUDA graph, then one timed
call), and the device RK45 solve of the probability-flow ODE (``get_ode_sampler``, rtol = atol = 1e-5) from the same
prior draw.  Each sampler run reports seconds per batch, images/s, milliseconds per step and the per-image rel-L2 of its
samples to the RK45 samples (max and median over the batch).  With random weights that distance is an accuracy proxy,
not a sample-quality figure.  The GPU's name and power limit, and the SM clock sampled by nvidia-smi during each timed
run, are read in the same process.

    python tools/bench_dpm_solver.py [--batch 1024] [--out PATH]

Prints one JSON line per run, then one JSON result line; ``--out`` also writes the result line to PATH.
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

from bench import ClockSampler   # noqa: E402
from bench_ddpm import gpu_identity   # noqa: E402


def per_image_rel(a, b):
  a, b = a.double().flatten(1), b.double().flatten(1)
  return (a - b).norm(dim=1) / b.norm(dim=1)


def timed(fn):
  clocks = ClockSampler(0)
  clocks.start()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return out, time.perf_counter() - t0, clocks.stop()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=1024)
  ap.add_argument('--steps', default='10,20,50')
  ap.add_argument('--orders', default='2,3')
  ap.add_argument('--forwards', type=int, default=20)
  ap.add_argument('--networks', default='ncsnpp_ve,ddpmpp_vp')
  ap.add_argument('--out', default=None)
  args = ap.parse_args()

  from score_sde_pytorch_b200 import configs, sampling, sde_lib
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  dev = torch.device('cuda:0')
  name, power = gpu_identity(0)
  B = args.batch
  shape = (B, 3, 32, 32)
  results = []
  for net in [n for n in args.networks.split(',') if n]:
    if net == 'ncsnpp_ve':
      cfg = configs.ve_cifar10_ncsnpp_continuous()
      sde = sde_lib.VESDE(cfg.model.sigma_min, cfg.model.sigma_max, cfg.model.num_scales)
    else:
      cfg = configs.vp_cifar10_ddpmpp_continuous()
      sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales)
    cfg.model.init_scale = 1.0     # init_scale = 0 would zero every block's last convolution
    torch.manual_seed(0)
    model = NCSNpp(cfg, precision='f16').to(dev)
    torch.manual_seed(1)
    z = sde.prior_sampling(shape).to(dev)

    with torch.no_grad():
      lab = torch.full((B,), 0.5 if net != 'ncsnpp_ve' else 1.0, device=dev)
      for _ in range(3):
        model(z, lab, labels_uniform=True)

      def forwards():
        for _ in range(args.forwards):
          model(z, lab, labels_uniform=True)
      _, wall, clk = timed(forwards)
    fwd_ms = 1e3 * wall / args.forwards
    print(json.dumps(dict(network=net, forward_ms=round(fwd_ms, 3), clocks=clk)), flush=True)

    ode = sampling.get_ode_sampler(sde, shape, lambda v: v, rtol=1e-5, atol=1e-5, eps=1e-3, device=dev)
    (x_rk, nfev), wall_rk, clk_rk = timed(lambda: ode(model, z=z.clone()))
    rk = dict(seconds_per_batch=round(wall_rk, 3), nfev=int(nfev), images_per_s=round(B / wall_rk, 2),
              solver=ode.last_stats['solver'], clocks=clk_rk)
    print(json.dumps(dict(network=net, rk45=rk)), flush=True)

    runs = []
    for order in [int(o) for o in args.orders.split(',')]:
      for steps in [int(s) for s in args.steps.split(',')]:
        fn = sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, steps=steps, order=order, eps=1e-3, device=dev)
        fn(model, z=z.clone())                                        # plan, graph capture
        (x, nfe), wall, clk = timed(lambda: fn(model, z=z.clone()))
        rel = per_image_rel(x, x_rk)
        r = dict(order=order, steps=steps, nfe=int(nfe), loop=fn.last_stats['loop'], seconds_per_batch=round(wall, 4),
                 images_per_s=round(B / wall, 1), ms_per_step=round(1e3 * wall / steps, 3),
                 rel_l2_to_rk45_max=float('%.3e' % rel.max()), rel_l2_to_rk45_median=float('%.3e' % rel.median()),
                 finite=bool(torch.isfinite(x).all()), clocks=clk)
        print(json.dumps(dict(network=net, run=r)), flush=True)
        runs.append(r)
    results.append(dict(network=net, forward_ms=round(fwd_ms, 3), forward_clocks=clk, rk45=rk, runs=runs))
    del model
    torch.cuda.empty_cache()

  line = dict(metric='multistep DPM-Solver++ sampling time per batch, CIFAR-10 32x32, f16, batch %d' % B, unit='s',
              higher_is_better=False, gpu=name, power_limit_w=power, batch=B, precision='f16', results=results,
              config=dict(algorithm='dpmsolver++', skip_type='logSNR', eps=1e-3, denoise=False,
                          networks='ncsnpp_ve: configs/ve/cifar10_ncsnpp_continuous.py, VESDE(0.01, 50); ddpmpp_vp: '
                                   'configs/vp/cifar10_ddpmpp_continuous.py, VPSDE(0.1, 20)',
                          weights='random init at init_scale 1, torch.manual_seed(0)',
                          prior='sde.prior_sampling, torch.manual_seed(1), the same draw for every run of a network',
                          reference='device RK45 solve of the probability-flow ODE, rtol = atol = 1e-5, same network',
                          sample_quality='not measured (FID needs data and Inception weights)'))
  text = json.dumps(line)
  print(text)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(text + '\n')


if __name__ == '__main__':
  main()
