#!/usr/bin/env python
"""Bits/dim with each explicit Runge-Kutta method of the device solver: DDPM cont. CIFAR-10
(``configs/vp/ddpm/cifar10_continuous.py``), VP SDE, tf32, batch 128, Rademacher, rtol = atol = 1e-5, eps = 1e-5 - the
setup of ``tools/bench_likelihood.py``, with the same weights, data and Hutchinson draw.

For ``method`` in RK23, RK45 and DOP853 it times one full ``likelihood.get_likelihood_fn(..., method=m)`` call on the
device-resident solve, and for one method (``--host-method``) the same call on the host loop (``device_solver=False``:
scipy's ``solve_ivp`` over the same engine evaluations, the whole state crossing PCIe twice per evaluation).  Each run
reports wall time, NFE, milliseconds per evaluation, device -> host reads and the mean bpd; the GPU's name, power limit and
SM clocks (sampled by nvidia-smi during each timed run) are read in the same process.

    python tools/bench_ode_methods.py [--methods RK23,RK45,DOP853] [--host-method RK45] [--out PATH]

Each run prints one JSON line as it finishes (``"run": ...``), then one JSON result line with all runs; ``--out`` also
writes the result line to PATH.  Writes nothing to the tree unless PATH points there.
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

METHODS = ('RK23', 'RK45', 'DOP853')


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=128)
  ap.add_argument('--precision', default='tf32', choices=['tf32', 'fp32'])
  ap.add_argument('--tol', type=float, default=1e-5)
  ap.add_argument('--methods', default=','.join(METHODS), help='comma-separated subset of ' + ','.join(METHODS))
  ap.add_argument('--host-method', default='RK45', choices=METHODS + ('none',))
  ap.add_argument('--out', default=None)
  args = ap.parse_args()

  from oracle import ddpm_oracle
  from score_sde_pytorch_b200 import configs, likelihood, sde_lib
  from score_sde_pytorch_b200.models.ddpm import DDPM
  dev = torch.device('cuda:0')
  cfg = configs.vp_cifar10_ddpm_continuous()
  torch.manual_seed(0)
  model = DDPM(cfg, precision=args.precision)
  model.load_state_dict(ddpm_oracle.redraw_zero_init(model.state_dict()))
  model = model.to(dev)
  sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales)
  g = torch.Generator().manual_seed(3)
  B = args.batch
  data = ((torch.randint(0, 256, (B, 3, 32, 32), generator=g).float() + torch.rand(B, 3, 32, 32, generator=g)) / 256.)
  data = (data * 2. - 1.).to(dev)
  torch.cuda.manual_seed(7)
  epsilon = torch.randint_like(data, low=0, high=2).float() * 2 - 1.     # likelihood_fn's own draw under this seed
  inverse_scaler = lambda x: (x + 1.) / 2.
  name, power = gpu_identity(0)

  with torch.no_grad():                                                  # build the tangent engine, warm its plan
    for _ in range(3):
      model.jvp(data, torch.full((B,), 500.0, device=dev), epsilon, labels_uniform=True)
  torch.cuda.synchronize()

  def run(method, device_solver):
    fn = likelihood.get_likelihood_fn(sde, inverse_scaler, rtol=args.tol, atol=args.tol, method=method,
                                      device_solver=device_solver)
    clocks = ClockSampler(0)
    clocks.start()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    bpd, z, nfe = fn(model, data, epsilon=epsilon)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    clk = clocks.stop()
    st = fn.last_stats
    r = dict(method=method, solver=st['solver'], wall_s=round(wall, 3), nfe=int(nfe),
             ms_per_eval=round(1e3 * wall / nfe, 3), host_reads=st.get('host_scalar_reads', 'not counted'),
             bpd_mean=round(float(bpd.mean()), 6), finite=bool(torch.isfinite(bpd).all() and torch.isfinite(z).all()),
             clocks=clk)
    print(json.dumps(dict(run=r)), flush=True)
    return r

  methods = [m for m in args.methods.split(',') if m]
  assert all(m in METHODS for m in methods), methods
  runs = [run(m, True) for m in methods]
  if args.host_method != 'none':
    runs.append(run(args.host_method, False))
  line = dict(metric='bits/dim wall time per method, DDPM cont. CIFAR-10 VP, rtol=atol=%g, Rademacher, batch %d' % (args.tol, B),
              unit='s', higher_is_better=False, gpu=name, power_limit_w=power, batch=B, precision=args.precision,
              runs=runs,
              config=dict(workload='configs/vp/ddpm/cifar10_continuous.py network (35.2 M parameters), 32x32',
                          weights='random init, zero-init weights re-drawn at scale 1, torch.manual_seed(0)',
                          data='uniformly dequantised random 8-bit images, torch.Generator seed 3, scaled to [-1, 1]',
                          hutchinson='Rademacher, torch.cuda.manual_seed(7), the same draw for every run'))
  text = json.dumps(line)
  print(text)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(text + '\n')


if __name__ == '__main__':
  main()
