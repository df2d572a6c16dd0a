#!/usr/bin/env python
"""Speed and accuracy of the engine's precision modes 'tf32', 'tf32x3' (split TF32) and 'fp32' (strict fp32, CUDA cores).

  * ms per evaluation (median of CUDA-event timings of single forwards) of NCSN++ cont. CIFAR-10 VE and DDPM++ cont.
    CIFAR-10 at batch 128 and 1024;
  * the bits/dim setup of tools/bench_likelihood.py (DDPM cont. CIFAR-10, VP, RK45, rtol = atol = 1e-5, Rademacher,
    batch 128): wall seconds, evaluations, mean bpd;
  * the error of one evaluation (batch 4) against a float64 run of the oracle network, per-image relative L2 (max).

Weights: the random init at init_scale 1 (NCSN++, DDPM++) or with the zero-initialised weights re-drawn at scale 1 (DDPM),
torch.manual_seed(0).  The GPU's name, power limit and SM clocks are read in the same run; no device setting is changed.

    python tools/bench_precision.py [--reps 5] [--skip-bpd]

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

from bench import ClockSampler   # noqa: E402
from bench_ddpm import gpu_identity   # noqa: E402

MODES = ('tf32', 'tf32x3', 'fp32')


def median_ms(fn, reps, warmup=2):
  for _ in range(warmup):
    fn()
  out = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    out.append(a.elapsed_time(b))
  return statistics.median(out)


def networks():
  from oracle import ddpm_oracle
  from score_sde_pytorch_b200 import configs
  from score_sde_pytorch_b200.models.ddpm import DDPM
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp

  def ve():
    c = configs.ve_cifar10_ncsnpp_continuous()
    c.model.init_scale = 1.0
    return c

  def ddpmpp():
    c = configs.vp_cifar10_ddpmpp_continuous()
    c.model.init_scale = 1.0
    return c

  def ddpm_model(precision):
    torch.manual_seed(0)
    m = DDPM(configs.vp_cifar10_ddpm_continuous(), precision=precision)
    m.load_state_dict(ddpm_oracle.redraw_zero_init(m.state_dict()))
    return m

  def ncsnpp_model(cfg_fn):
    def make(precision):
      torch.manual_seed(0)
      return NCSNpp(cfg_fn(), precision=precision)
    return make

  return {'ncsnpp_cifar10_ve': (ncsnpp_model(ve), 'sigma'), 'ddpmpp_cifar10': (ncsnpp_model(ddpmpp), 't'),
          'ddpm_cifar10': (ddpm_model, 't')}


def labels_for(kind, B, dev):
  g = torch.Generator().manual_seed(5)
  if kind == 'sigma':
    return (0.01 * (50 / 0.01) ** torch.rand(B, generator=g)).to(dev)
  return (torch.rand(B, generator=g) * 999.).to(dev)


def float64_oracle(name, sd, cfg, x, labels):
  from oracle import ddpm_oracle as DO, ncsnpp_oracle as NO
  up, te = NO.upfirdn2d_native, NO.timestep_embedding
  te64 = lambda t, dim, **kw: te(t, dim, **kw).double()
  NO.upfirdn2d_native, NO.timestep_embedding, DO.timestep_embedding = (lambda v, k, **kw: up(v, k.to(v.dtype), **kw)), te64, te64
  try:
    fwd = DO.ddpm_forward if name == 'ddpm_cifar10' else NO.ncsnpp_forward
    with torch.no_grad():
      return fwd({k: v.double() for k, v in sd.items()}, cfg, x.double(), labels.double())
  finally:
    NO.upfirdn2d_native, NO.timestep_embedding, DO.timestep_embedding = up, te, te


def rel_l2(a, b):
  a, b = a.double().flatten(1), b.double().flatten(1)
  return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=5)
  ap.add_argument('--skip-bpd', action='store_true')
  args = ap.parse_args()
  dev = torch.device('cuda:0')
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  name, power = gpu_identity(0)
  nets = networks()
  clocks = ClockSampler(0)
  clocks.start()

  speed, error = {}, {}
  for net, (make, kind) in nets.items():
    g = torch.Generator().manual_seed(9)
    x4 = torch.randn(4, 3, 32, 32, generator=g).to(dev)
    l4 = labels_for(kind, 4, dev)
    ys, sd, cfg = {}, None, None
    for mode in MODES:
      model = make(mode).to(dev)
      sd, cfg = model.state_dict(), model.config
      with torch.no_grad():
        ys[mode] = model(x4, l4)
        if net != 'ddpm_cifar10':
          for B in (128, 1024):
            x = torch.randn(B, 3, 32, 32, generator=g).to(dev)
            lab = labels_for(kind, B, dev)
            speed.setdefault(net, {}).setdefault(f'batch{B}', {})[mode] = round(median_ms(lambda: model(x, lab), args.reps), 3)
      model._release()
      del model
      torch.cuda.empty_cache()
    ref = float64_oracle(net, sd, cfg, x4, l4)
    error[net] = {m: float(f'{rel_l2(y, ref):.3e}') for m, y in ys.items()}

  bpd = {}
  if not args.skip_bpd:
    from score_sde_pytorch_b200 import likelihood, sde_lib
    from score_sde_pytorch_b200 import configs
    cfg = configs.vp_cifar10_ddpm_continuous()
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales)
    g = torch.Generator().manual_seed(3)
    B = 128
    data = ((torch.randint(0, 256, (B, 3, 32, 32), generator=g).float() + torch.rand(B, 3, 32, 32, generator=g)) / 256.)
    data = (data * 2. - 1.).to(dev)
    for mode in MODES:
      model = nets['ddpm_cifar10'][0](mode).to(dev)
      fn = likelihood.get_likelihood_fn(sde, lambda v: (v + 1.) / 2.)
      torch.cuda.manual_seed(7)
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      b, _, nfe = fn(model, data)
      torch.cuda.synchronize()
      bpd[mode] = dict(wall_s=round(time.perf_counter() - t0, 3), nfe=int(nfe), bpd_mean=round(float(b.mean()), 6),
                       solver=fn.last_stats.get('solver'))
      model._release()
      del model
      torch.cuda.empty_cache()
  clk = clocks.stop()

  print(json.dumps(dict(
      metric='ms per evaluation by precision mode (median of CUDA-event timings), NCSN++ cont. CIFAR-10 VE / DDPM++ cont. '
             'CIFAR-10; bits/dim of DDPM cont. CIFAR-10 (RK45, rtol=atol=1e-5, batch 128); one-evaluation rel-L2 vs a '
             'float64 oracle run',
      gpu=name, power_limit_w=power, clocks=clk, ms_per_eval=speed, bits_per_dim=bpd or 'not measured',
      rel_l2_vs_float64_oracle=error, reps=args.reps,
      config=dict(weights='random init, init_scale 1 (NCSN++, DDPM++) / zero-init weights re-drawn at scale 1 (DDPM), '
                          'torch.manual_seed(0)',
                  data='random normal inputs; bits/dim: uniformly dequantised random 8-bit images, torch.Generator seed 3'))))


if __name__ == '__main__':
  main()
