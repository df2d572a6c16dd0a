#!/usr/bin/env python
"""NCSNv2 on the engine: the CIFAR-10 network of ``configs/ve/ncsnv2/cifar10.py`` (``ncsnv2_64``, nf=128, 29.7 M
parameters, 32x32).

  * ms per network evaluation at batch 128 and 1024 in tf32 and f16 (CUDA events around `--evals` back-to-back forwards
    after `--warmup`), and the same forward through the plain-PyTorch oracle (oracle/ncsnv2_oracle.py, eager, fp32 with
    PyTorch's default cuDNN settings) on the same GPU as the baseline;
  * images/s of the config's sampler (predictor 'none', annealed Langevin dynamics with 5 steps per noise level,
    continuous=False, the host loop over the engine network) at batch 1024: `--levels` noise levels are timed after one
    warm-up level and the rate is extrapolated to the config's 232 levels.

Weights are the random init under ``torch.manual_seed(0)``, data synthetic.  The GPU's name and enforced power limit
are read in the same run.  One JSON document on stdout, and in `--out` when given:

    python tools/bench_ncsnv2.py --out records/bench_cifar10_ncsnv2_h100.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from bench import ClockSampler   # noqa: E402


def gpu_identity(index):
  name = torch.cuda.get_device_name(index)
  try:
    out = subprocess.run(['nvidia-smi', f'--id={index}', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    power, sm_max = (float(v) for v in out.splitlines()[0].split(','))
  except (OSError, ValueError, IndexError, subprocess.SubprocessError):
    power, sm_max = None, None
  return name, power, sm_max


def time_ms(fn, warmup, reps):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--evals', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--levels', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()

  from oracle import ncsnv2_oracle
  from score_sde_pytorch_b200 import configs, sampling, sde_lib
  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2
  dev = torch.device('cuda:0')
  cfg = configs.ve_cifar10_ncsnv2()
  name, power, sm_max = gpu_identity(0)
  clocks = ClockSampler(0)
  clocks.start()
  forward = {}
  models = {}
  for precision in ('tf32', 'f16'):
    torch.manual_seed(0)
    models[precision] = NCSNv2(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in models['tf32'].state_dict().items()}
  for batch in (128, 1024):
    torch.manual_seed(1)
    x = torch.rand(batch, 3, 32, 32, device=dev)
    y = torch.randint(0, cfg.model.num_scales, (batch,), device=dev)
    row = {}
    with torch.no_grad():
      for precision, model in models.items():
        row[f'engine_{precision}_ms'] = round(time_ms(lambda: model(x, y), args.warmup, args.evals), 3)
      row['oracle_fp32_eager_ms'] = round(time_ms(lambda: ncsnv2_oracle.ncsnv2_forward(sd, cfg, x, y), 1, max(2, args.evals // 2)), 3)
    for precision in models:
      row[f'speedup_{precision}_vs_oracle'] = round(row['oracle_fp32_eager_ms'] / row[f'engine_{precision}_ms'], 2)
    forward[f'batch_{batch}'] = row
  # the config's sampler on the host loop: corrector_update_fn is the loop body of sampling.get_pc_sampler
  sde = sde_lib.VESDE(sigma_min=cfg.model.sigma_min, sigma_max=cfg.model.sigma_max, N=cfg.model.num_scales)
  model = models['tf32']
  B = 1024
  torch.manual_seed(2)
  x = sde.prior_sampling((B, 3, 32, 32)).to(dev)
  timesteps = torch.linspace(sde.T, 1e-5, sde.N, device=dev)

  def level(i, x):
    vec_t = torch.ones(B, device=dev) * timesteps[i]
    return sampling.shared_corrector_update_fn(x, vec_t, sde=sde, model=model, corrector=sampling.AnnealedLangevinDynamics,
                                               continuous=False, snr=cfg.sampling.snr, n_steps=cfg.sampling.n_steps_each)[0]

  with torch.no_grad():
    x = level(0, x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(1, 1 + args.levels):
      x = level(i, x)
    e1.record()
    torch.cuda.synchronize()
  ms_level = e0.elapsed_time(e1) / args.levels
  clk = clocks.stop()
  rec = dict(
      gpu=name, power_limit_w=power, sm_max_mhz=sm_max,
      command='python tools/bench_ncsnv2.py ' + ' '.join(sys.argv[1:]),
      network='configs/ve/ncsnv2/cifar10.py (ncsnv2_64, nf=128, 29.7 M parameters, 32x32)',
      forward_ms_per_evaluation=forward,
      sampler=dict(metric='ALD sampler images/s, CIFAR-10 NCSNv2 (232 levels x 5 Langevin steps, host loop, tf32)',
                   batch=B, levels_timed=args.levels, ms_per_level=round(ms_level, 3),
                   images_per_s=round(B / (sde.N * ms_level / 1e3), 4), finite=bool(torch.isfinite(x).all()),
                   state_dtype=str(x.dtype)),
      clocks=clk, evals=args.evals, warmup=args.warmup,
      weights='random init, torch.manual_seed(0)', data='synthetic')
  txt = json.dumps(rec, indent=1)
  print(txt)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(txt + '\n')


if __name__ == '__main__':
  main()
