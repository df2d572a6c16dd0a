#!/usr/bin/env python
"""Inpainting and colorization: the native PC loop against the host loop, on the network ``bench.py`` measures
(``configs/ve/cifar10_ncsnpp_continuous.py``, ``model.init_scale = 1``, random init under ``torch.manual_seed(0)``,
fp16 tensor-core operands), VE SDE, reverse diffusion + Langevin, snr 0.16, one corrector step.

Both loops run through ``controllable_generation.get_pc_inpainter`` / ``get_pc_colorizer`` on the same engine: the
stock classes select the native loop, a trivial subclass of ``LangevinCorrector`` the host loop (two engine forwards
enqueued from the host plus the eager-torch blend per iteration).  The SDE has ``N = --steps`` discretisation steps, so
one call is ``--steps`` PC iterations; the per-iteration cost does not depend on N.  Per batch size and task: one
warm-up call of each loop, then ``--reps`` timed calls of each, alternating host and native, each bracketed by a device
synchronise.  Reported: median ms per iteration of each loop, their ratio, and the per-image relative L2 between the
two loops' outputs under the same seeds.  Data are seeded random images; the inpainting mask keeps the left half.
The GPU's name and power limit are read in the same run.

    python tools/bench_controllable.py [--batches 1024 8] [--steps 10] [--reps 3]

One JSON line on stdout.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_ddpm import gpu_identity   # noqa: E402


def rel_l2(a, b):
  a, b = a.double().flatten(1), b.double().flatten(1)
  return ((a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-30)).max().item()


def timed(fn, *args):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn(*args)
  torch.cuda.synchronize()
  return time.perf_counter() - t0, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batches', type=int, nargs='+', default=[1024, 8])
  ap.add_argument('--steps', type=int, default=10, help='PC iterations per call (the SDE\'s N)')
  ap.add_argument('--reps', type=int, default=3, help='timed calls per loop, alternating')
  ap.add_argument('--precision', default='f16', choices=['f16', 'tf32', 'fp32'])
  args = ap.parse_args()

  from score_sde_pytorch_b200 import configs, controllable_generation as CG, sampling, sde_lib
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  dev = torch.device('cuda:0')
  torch.backends.cuda.matmul.allow_tf32 = False   # the host loop's colour transform runs in fp32, as in the reference
  cfg = configs.ve_cifar10_ncsnpp_continuous()
  cfg.model.init_scale = 1.0
  torch.manual_seed(0)
  model = NCSNpp(cfg, precision=args.precision).to(dev)
  sde = sde_lib.VESDE(0.01, 50, args.steps)
  name, power = gpu_identity(0)

  class HostLangevin(sampling.LangevinCorrector):   # not a stock class: the host loop runs
    pass

  kw = dict(snr=0.16, n_steps=1, probability_flow=False, continuous=True, denoise=True, eps=1e-5)
  results = []
  for B in args.batches:
    g = torch.Generator().manual_seed(3)
    data = torch.rand(B, 3, 32, 32, generator=g).to(dev)
    mask = torch.zeros(B, 1, 32, 32, device=dev)
    mask[..., :16] = 1.
    gray = data.mean(1, keepdim=True).expand(B, 3, 32, 32).contiguous()
    for task in ('inpaint', 'colorize'):
      make = CG.get_pc_inpainter if task == 'inpaint' else CG.get_pc_colorizer
      fns = dict(native=make(sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, lambda v: v, **kw),
                 host=make(sde, sampling.ReverseDiffusionPredictor, HostLangevin, lambda v: v, **kw))
      inputs = (data, mask) if task == 'inpaint' else (gray,)
      outs, times = {}, {k: [] for k in fns}
      for k, fn in fns.items():   # warm-up: engine plan, graph capture, allocator
        torch.manual_seed(5); torch.cuda.manual_seed(5)
        timed(fn, model, *inputs)
      for _ in range(args.reps):
        for k in ('host', 'native'):
          torch.manual_seed(5); torch.cuda.manual_seed(5)
          dt, out = timed(fns[k], model, *inputs)
          times[k].append(dt * 1e3 / args.steps)
          outs[k] = out
          assert fns[k].last_stats['loop'] == k, (k, fns[k].last_stats)
      host, nat = statistics.median(times['host']), statistics.median(times['native'])
      results.append(dict(batch=B, task=task, host_ms_per_iter=round(host, 3), native_ms_per_iter=round(nat, 3),
                          host_over_native=round(host / nat, 4),
                          host_ms_all=[round(t, 3) for t in times['host']],
                          native_ms_all=[round(t, 3) for t in times['native']],
                          rel_l2_native_vs_host=float('%.3g' % rel_l2(outs['native'], outs['host'])),
                          finite=bool(torch.isfinite(outs['native']).all()),
                          launches_per_iter=fns['native'].last_stats['launches_per_step']))
      print(json.dumps(results[-1]), file=sys.stderr, flush=True)

  print(json.dumps(dict(
      metric='controllable generation, ms per PC iteration, native loop vs host loop',
      gpu=name, power_limit_w=power, precision=args.precision, steps_per_call=args.steps, reps=args.reps,
      results=results,
      config=dict(workload='configs/ve/cifar10_ncsnpp_continuous.py network, 32x32, VE SDE (sigma 0.01..50), '
                           'reverse_diffusion + langevin, snr 0.16, n_steps_each 1, denoise',
                  weights='random init, init_scale=1, torch.manual_seed(0)',
                  data='torch.rand images (Generator seed 3); inpainting keeps the left half; colorization gets the '
                       'channel mean',
                  timing='host clock around each call, device-synchronised; warm-up call of each loop first; '
                         'host and native alternate'))))


if __name__ == '__main__':
  main()
