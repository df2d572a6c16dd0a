#!/usr/bin/env python
"""Sampling throughput of the DDPM network: DDPM cont. CIFAR-10 (``configs/vp/ddpm/cifar10_continuous.py``), VP SDE with
1000 steps, Euler-Maruyama predictor and no corrector (the config's own sampler), batch 1024, fp16 tensor-core operands.

A step is one PC iteration over the batch (one network evaluation plus the predictor update with in-kernel noise),
replayed as one CUDA graph by the native loop, timed with CUDA events; images/s = batch / (1000 * seconds per step).
Weights are the random init with the zero-initialised weights re-drawn at scale 1 (so activations have their trained
magnitudes), ``torch.manual_seed(0)``.  The GPU's name and enforced power limit are read in the same run and printed
beside the result, since both are part of the number.

    python tools/bench_ddpm.py --steps 20 --warmup 3

One JSON line on stdout.  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from bench import ClockSampler, timed_steps   # noqa: E402

N_SAMPLER_STEPS = 1000


def gpu_identity(index):
  name = torch.cuda.get_device_name(index)
  try:
    out = subprocess.run(['nvidia-smi', f'--id={index}', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    power = float(out.splitlines()[0])
  except (OSError, ValueError, IndexError, subprocess.SubprocessError):
    power = None
  return name, power


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--batch', type=int, default=1024)
  ap.add_argument('--precision', default='f16', choices=['f16', 'tf32', 'fp32'])
  args = ap.parse_args()

  from oracle import ddpm_oracle
  from score_sde_pytorch_b200 import configs, native, sampling, sde_lib
  from score_sde_pytorch_b200.models.ddpm import DDPM
  dev = torch.device('cuda:0')
  cfg = configs.vp_cifar10_ddpm_continuous()
  torch.manual_seed(0)
  model = DDPM(cfg, precision=args.precision)
  model.load_state_dict(ddpm_oracle.redraw_zero_init(model.state_dict()))
  model = model.to(dev)
  sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, N_SAMPLER_STEPS)
  shape = (args.batch, 3, 32, 32)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.EulerMaruyamaPredictor,
                              corrector=sampling.NoneCorrector, shape=shape, snr=cfg.sampling.snr, n_steps=1,
                              probability_flow=False, continuous=True, eps=1e-3, device=dev)
  assert plan is not None, 'the native PC loop does not cover this sampler'
  torch.manual_seed(1)
  x0 = sde.prior_sampling(shape).to(dev)
  name, power = gpu_identity(0)
  clocks = ClockSampler(0)
  clocks.start()
  ms = timed_steps(plan, x0, args.warmup, args.steps)
  clk = clocks.stop()
  finite = bool(torch.isfinite(plan._x).all())
  print(json.dumps(dict(
      metric='PC-sampler images/sec, DDPM cont. CIFAR-10 1000-step VP (Euler-Maruyama, no corrector)',
      value=round(args.batch / (N_SAMPLER_STEPS * ms / 1e3), 4), unit='images/s', higher_is_better=True,
      gpu=name, power_limit_w=power, batch=args.batch, precision=args.precision, steps=args.steps, warmup=args.warmup,
      ms_per_step=round(ms, 4), launches_per_forward=model.launches_per_forward(),
      launches_per_step=plan.launches_per_step(), clocks=clk, finite=finite,
      config=dict(workload='configs/vp/ddpm/cifar10_continuous.py network (35.2 M parameters), 32x32',
                  step='one PC iteration = Euler-Maruyama predictor (1 score evaluation)',
                  weights='random init, zero-init weights re-drawn at scale 1, torch.manual_seed(0)', data='synthetic'))))


if __name__ == '__main__':
  main()
