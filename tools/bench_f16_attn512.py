#!/usr/bin/env python
"""'f16' against 'tf32' on the networks with 512-channel attention at 16x16 (T = 256 tokens, C = 512 channels).

  * ms per evaluation (median of CUDA-event timings of single forwards after warm-up) of DDPM CelebA-HQ-256
    (configs/vp/ddpm/celebahq.py) at batch 1, 8, 32 and of NCSN++ FFHQ-1024 (configs/ve/ffhq_ncsnpp_continuous.py) at
    batch 1, 2, in 'tf32' and 'f16';
  * one 16x16, 512-channel attention core in isolation at batch 1, 8, 64: the fused f16 kernel (logits, softmax, P.V,
    NIN_3, residual, quad sums) against the three tensor-core contractions of the tf32 chain (Q K^T, P V, O W3^T; its
    softmax launch is not included, so the tf32 figure is a lower bound for that chain);
  * per-image relative L2 of one f16 and one tf32 evaluation at batch 1 against the strict-fp32 oracle on the same inputs.

Weights: random init, init_scale 1 (NCSN++) / zero-initialised weights re-drawn at scale 1 (DDPM), torch.manual_seed(0).
The GPU's name, power limit and SM clocks are read in the same run; no device setting is changed.

    python tools/bench_f16_attn512.py [--reps 10] [--out FILE.json]

One JSON line on stdout (and in --out when given).
"""
import argparse
import json
import os
import statistics
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (REPO, os.path.join(REPO, 'tests'), os.path.dirname(os.path.abspath(__file__))):
  if _p not in sys.path:
    sys.path.insert(0, _p)

from bench import ClockSampler           # noqa: E402
from bench_ddpm import gpu_identity      # noqa: E402

MODES = ('tf32', 'f16')


def median_ms(fn, reps, warmup=3):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  out = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    out.append(a.elapsed_time(b))
  return statistics.median(out)


def rel_l2(a, b):
  a, b = a.double().flatten(1), b.double().flatten(1)
  return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item()


def make_network(name, precision):
  from oracle import ddpm_oracle
  from score_sde_pytorch_b200 import configs
  from score_sde_pytorch_b200.models.ddpm import DDPM
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  torch.manual_seed(0)
  if name == 'ddpm_celebahq_256':
    m = DDPM(configs.vp_celebahq_256_ddpm(), precision=precision)
    m.load_state_dict(ddpm_oracle.redraw_zero_init(m.state_dict()))
    return m
  c = configs.ve_ffhq_1024_ncsnpp_continuous()
  c.model.init_scale = 1.0
  return NCSNpp(c, precision=precision)


NETWORKS = {'ddpm_celebahq_256': (256, (1, 8, 32)), 'ncsnpp_ffhq_1024': (1024, (1, 2))}


def inputs(name, B, R, dev):
  g = torch.Generator().manual_seed(100 + B)
  x = torch.randn(B, 3, R, R, generator=g)
  if name == 'ddpm_celebahq_256':
    return x.to(dev), (torch.rand(B, generator=g) * 999.).to(dev)
  return (x * 5).to(dev), (0.01 * (348 / 0.01) ** torch.rand(B, generator=g)).to(dev)


def oracle(name, model, x, labels):
  from oracle import ddpm_oracle as DO, ncsnpp_oracle as NO
  sd = {k: v.to(x.device) for k, v in model.state_dict().items()}
  fwd = DO.ddpm_forward if name == 'ddpm_celebahq_256' else NO.ncsnpp_forward
  with torch.no_grad():
    return fwd(sd, model.config, x, labels)


def attention_core_timings(reps, dev):
  import gpu_util
  T, C = 256, 512
  out = {}
  for nimg in (1, 8, 64):
    g = torch.Generator().manual_seed(nimg)
    qk = (torch.randn(nimg * T, 2 * C, generator=g) * 1.5).to(dev)
    vT = torch.randn(nimg, C, T, generator=g).to(dev)
    w3 = (torch.randn(C, C, generator=g) / 22).to(dev)
    bv, b3 = torch.randn(C, generator=g).to(dev), torch.randn(C, generator=g).to(dev)
    x = torch.randn(nimg * T, C, generator=g).to(dev)
    qk16, vT16, w316 = qk.half(), vT.half(), w3.half()
    fused = median_ms(lambda: gpu_util.attention_core(qk16, vT16, w316, bv, b3, x, 0.7071067690849304), reps)
    qkt, vTt, w3t = gpu_util.round_tf32(qk), gpu_util.round_tf32(vT), gpu_util.round_tf32(w3)
    P = gpu_util.round_tf32(torch.softmax(torch.randn(nimg * T, T, generator=g), -1).to(dev))
    O = gpu_util.round_tf32(torch.randn(nimg * T, C, generator=g).to(dev))

    def chain():
      gpu_util.gemm_nt(qkt, qkt[:, C:], nimg, T, T, C, lda=2 * C, ldw=2 * C, impl=1)          # S = Q K^T
      gpu_util.gemm_nt(P, vTt, nimg, T, C, T, impl=1)                                          # O = P V
      gpu_util.gemm_nt(O, w3t, 1, nimg * T, C, C, bias=b3, impl=1)                             # Y = O W3^T
    tf32 = median_ms(chain, reps)
    out[f'batch{nimg}'] = dict(fused_f16_ms=round(fused, 4), tf32_contractions_ms=round(tf32, 4))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=10)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'bench_f16_attn512 needs a CUDA device'
  dev = torch.device('cuda:0')
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  name, power = gpu_identity(0)
  clocks = ClockSampler(0)
  clocks.start()
  speed, error = {}, {}
  for net, (R, batches) in NETWORKS.items():
    for mode in MODES:
      model = make_network(net, mode).to(dev)
      with torch.no_grad():
        for B in batches:
          x, lab = inputs(net, B, R, dev)
          speed.setdefault(net, {}).setdefault(f'batch{B}', {})[mode] = round(median_ms(lambda: model(x, lab), args.reps), 3)
        x, lab = inputs(net, 1, R, dev)
        y = model(x, lab)
      error.setdefault(net, {})[mode] = float(f'{rel_l2(y, oracle(net, model, x, lab)):.3e}')
      model._release()
      del model
      torch.cuda.empty_cache()
  for net in speed:
    for b in speed[net].values():
      b['f16_over_tf32'] = round(b['f16'] / b['tf32'], 3)
  core = attention_core_timings(args.reps, dev)
  clk = clocks.stop()
  rec = dict(
      metric="ms per evaluation in 'tf32' and 'f16' (median of CUDA-event timings), the 16x16 512-channel attention core "
             "in isolation, and one-evaluation per-image rel-L2 vs the strict-fp32 oracle at batch 1",
      gpu=name, power_limit_w=power, clocks=clk, ms_per_eval=speed, attention_core_T256_C512=core,
      rel_l2_vs_fp32_oracle=error, reps=args.reps,
      config=dict(weights='random init, init_scale 1 (NCSN++) / zero-init weights re-drawn at scale 1 (DDPM), torch.manual_seed(0)',
                  data='random normal images (x5 for NCSN++), random time labels / log-uniform sigmas'))
  line = json.dumps(rec)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(line + '\n')


if __name__ == '__main__':
  main()
