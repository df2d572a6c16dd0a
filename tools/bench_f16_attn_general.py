#!/usr/bin/env python
"""The flash fp16 attention core (csrc/attn_flash.cu) against the tf32 chain it replaces in 'f16' plans, and 'f16'
against 'tf32' on whole networks whose attention runs on it.

  * the attention block without its q / k / v projections, at (T, C) in (256, 128), (1024, 128), (1024, 256),
    (1024, 512), (4096, 128) and batch 1, 8, 64:
      f16  = flash core (Q K^T, online softmax, P V + b_v) + the NIN_3 contraction (fp16 operands), as the f16 plan runs it;
      tf32 = S = Q K^T, row softmax, O = P V + b_v, NIN_3 (three TF32 tensor-core contractions and one softmax launch,
             the logits through HBM), as the tf32 plan runs it (T <= 1024: the row softmax has no longer rows);
    each figure is the median over reps of one CUDA-graph replay of 10 back-to-back block evaluations (CUDA events),
    divided by 10, after warm-up.  The flash core is also timed alone; its achieved FLOP/s (4 B T^2 C operations) and
    its share of the H100 SXM data-sheet bound are reported: the larger of the FLOP time at 989 TFLOP/s dense fp16 and
    the byte time (q, k, v^T read once, O written once) at 3.35 TB/s, with the bound that applies named;
  * ms per evaluation (median of CUDA-event timings of single forwards after warm-up) of the three test networks at
    batch 128 in 'tf32' and 'f16';
  * accuracy of what was timed: per-image rel-L2 of the timed f16 and tf32 block outputs against the block computed in
    strict fp32 from the same operands, and of one f16 / tf32 network evaluation against the strict-fp32 oracle.

Weights: random init at torch.manual_seed(0) (NCSN++ init_scale 1; DDPM zero-init weights re-drawn at scale 1).  The
GPU's name, power limit and SM clocks are read in the same run; no device setting is changed.

    python tools/bench_f16_attn_general.py [--reps 20] [--out records/bench_f16_attn_general_h100.json]

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

PEAK_F16 = 989e12    # H100 SXM data sheet, dense fp16, 700 W card
PEAK_HBM = 3.35e12   # H100 SXM data sheet, HBM3 bytes/s
SHAPES = ((256, 128), (1024, 128), (1024, 256), (1024, 512), (4096, 128))
BATCHES = (1, 8, 64)
INNER = 10           # block evaluations per graph replay
SOFTMAX_MAX_T = 1024  # longest row of b200_softmax_rows_f32: the tf32 chain exists up to T = 1024


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


def graph_ms(fn, reps):
  """ms per call of fn: median over reps of one replay of a CUDA graph holding INNER calls (no host gaps)."""
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(INNER):
      fn()
  return median_ms(g.replay, reps) / INNER


def rel_l2_rows(a, b, nimg):
  a, b = a.double().reshape(nimg, -1), b.double().reshape(nimg, -1)
  return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item()


def block_timings(reps, dev):
  import gpu_util
  from score_sde_pytorch_b200 import _lib
  out = {}
  for T, C in SHAPES:
    for nimg in BATCHES:
      g = torch.Generator().manual_seed(T + C + nimg)
      qk = (torch.randn(nimg * T, 2 * C, generator=g) * 1.5).to(dev)
      vT = torch.randn(nimg, C, T, generator=g).to(dev)
      w3 = (torch.randn(C, C, generator=g) / C ** 0.5).to(dev)
      bv, b3 = torch.randn(C, generator=g).to(dev), torch.randn(C, generator=g).to(dev)
      qk16, vT16, w316 = qk.half(), vT.half(), w3.half()
      O16 = torch.empty(nimg * T, C, device=dev, dtype=torch.float16)
      Y16 = {}

      def flash():
        _lib.call('b200_attention_flash_f16', _lib.ptr(qk16), _lib.ptr(vT16), _lib.ptr(bv), _lib.ptr(O16), nimg, T, C,
                  _lib.stream_ptr(dev))

      def f16_block():
        flash()
        Y16['y'] = gpu_util.gemm_nt(O16, w316, 1, nimg * T, C, C, bias=b3, impl=2)                  # NIN_3

      qkt, vTt, w3t = gpu_util.round_tf32(qk), gpu_util.round_tf32(vT), gpu_util.round_tf32(w3)
      S = torch.empty(nimg * T, T, device=dev)
      Yt = {}

      def tf32_block():
        s = gpu_util.gemm_nt(qkt, qkt[:, C:], nimg, T, T, C, lda=2 * C, ldw=2 * C, impl=1)          # S = Q K^T
        _lib.call('b200_softmax_rows_f32', _lib.ptr(s), _lib.ptr(S), nimg * T, T, C ** -0.5, 1, _lib.stream_ptr(dev))
        o = gpu_util.gemm_nt(S, vTt, nimg, T, C, T, bias=bv, round_out=True, impl=1)                # O = P V + b_v
        Yt['y'] = gpu_util.gemm_nt(o, w3t, 1, nimg * T, C, C, bias=b3, impl=1)                      # NIN_3

      t_flash = graph_ms(flash, reps)
      t_f16 = graph_ms(f16_block, reps)
      t_tf32 = graph_ms(tf32_block, reps) if T <= SOFTMAX_MAX_T else None
      # the block in strict fp32 from the f16 operands (the tf32 operands differ from them by < 2^-11 relative)
      q = qk16[:, :C].float().reshape(nimg, T, C)
      k = qk16[:, C:].float().reshape(nimg, T, C)
      ref_o = torch.empty(nimg, T, C, device=dev)
      for i in range(nimg):
        ref_o[i] = torch.softmax((q[i] @ k[i].t()) * C ** -0.5, -1) @ vT16[i].float().t() + bv
      ref_y = ref_o.reshape(nimg * T, C) @ w316.float().t() + b3
      flops = 4.0 * nimg * T * T * C
      bytes_ = 8.0 * nimg * T * C
      t_min = max(flops / PEAK_F16, bytes_ / PEAK_HBM)
      out[f'T{T}_C{C}_batch{nimg}'] = dict(
          flash_ms=round(t_flash, 4), f16_block_ms=round(t_f16, 4),
          tf32_block_ms=round(t_tf32, 4) if t_tf32 else f'not available: the row softmax covers T <= {SOFTMAX_MAX_T}',
          f16_over_tf32=round(t_f16 / t_tf32, 3) if t_tf32 else None,
          flash_tflops=round(flops / (t_flash * 1e-3) / 1e12, 1),
          flash_share_of_bound=round(t_min / (t_flash * 1e-3), 3),
          bound='fp16 tensor FLOPs' if flops / PEAK_F16 >= bytes_ / PEAK_HBM else 'HBM bytes',
          rel_l2_flash_O=float(f'{rel_l2_rows(O16.float(), ref_o, nimg):.3e}'),
          rel_l2_f16_block=float(f'{rel_l2_rows(Y16["y"], ref_y, nimg):.3e}'),
          rel_l2_tf32_block=float(f'{rel_l2_rows(Yt["y"], ref_y, nimg):.3e}') if t_tf32 else None)
      print(f'T={T} C={C} batch {nimg}: {out[f"T{T}_C{C}_batch{nimg}"]}', file=sys.stderr)
      del S, qk, vT, qkt, vTt, Y16, Yt
      torch.cuda.empty_cache()
  return out


NETWORKS = {
    'A_ddpmpp_T256_C128': 'tiny_ddpmpp(nf=64, image_size=32, ch_mult=(1, 2, 2), attn_resolutions=(16,))',
    'B_ncsnpp_T1024_C128': 'tiny_ncsnpp(nf=64, image_size=32, ch_mult=(2, 4), attn_resolutions=(32,))',
    'C_ddpm_T1024_C128': 'tiny_ddpm(nf=64, image_size=64, ch_mult=(1, 2, 2, 2), attn_resolutions=(32,))',
}


def make_network(name, precision):
  from oracle import ddpm_oracle
  from score_sde_pytorch_b200 import configs
  from score_sde_pytorch_b200.models.ddpm import DDPM
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  torch.manual_seed(0)
  if name == 'A_ddpmpp_T256_C128':
    cfg = configs.tiny_ddpmpp(nf=64, image_size=32, ch_mult=(1, 2, 2), attn_resolutions=(16,))
  elif name == 'B_ncsnpp_T1024_C128':
    cfg = configs.tiny_ncsnpp(nf=64, image_size=32, ch_mult=(2, 4), attn_resolutions=(32,))
  else:
    m = DDPM(configs.tiny_ddpm(nf=64, image_size=64, ch_mult=(1, 2, 2, 2), attn_resolutions=(32,)), precision=precision)
    m.load_state_dict(ddpm_oracle.redraw_zero_init(m.state_dict()))
    return m
  cfg.model.init_scale = 1.0
  return NCSNpp(cfg, precision=precision)


def network_inputs(name, model, B, dev):
  R = model.config.data.image_size
  g = torch.Generator().manual_seed(100 + B)
  x = torch.randn(B, 3, R, R, generator=g)
  if model.config.training.sde == 'vesde':
    return (x * 5).to(dev), (0.01 * (50 / 0.01) ** torch.rand(B, generator=g)).to(dev)
  return x.to(dev), (torch.rand(B, generator=g) * 999.).to(dev)


def network_timings(reps, dev, batch=128):
  from oracle import ddpm_oracle as DO, ncsnpp_oracle as NO
  speed, error = {}, {}
  for name in NETWORKS:
    for mode in ('tf32', 'f16'):
      model = make_network(name, mode).to(dev)
      with torch.no_grad():
        x, lab = network_inputs(name, model, batch, dev)
        speed.setdefault(name, {})[mode] = round(median_ms(lambda: model(x, lab), reps), 3)
        y = model(x[:4], lab[:4])
        sd = {k: v.to(dev) for k, v in model.state_dict().items()}
        fwd = DO.ddpm_forward if name.startswith('C_') else NO.ncsnpp_forward
        ref = fwd(sd, model.config, x[:4], lab[:4])
      error.setdefault(name, {})[mode] = float(f'{rel_l2_rows(y, ref, 4):.3e}')
      if mode == 'f16':
        assert any('attention flash' in n for n in model.op_names())
      model._release()
      del model
      torch.cuda.empty_cache()
    speed[name]['f16_over_tf32'] = round(speed[name]['f16'] / speed[name]['tf32'], 3)
  return speed, error


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'bench_f16_attn_general needs a CUDA device'
  dev = torch.device('cuda:0')
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  name, power = gpu_identity(0)
  clocks = ClockSampler(0)
  clocks.start()
  blocks = block_timings(args.reps, dev)
  speed, error = network_timings(args.reps, dev)
  clk = clocks.stop()
  rec = dict(
      metric="attention block without projections: flash f16 core (+ NIN_3) vs the tf32 chain, ms per block (median of "
             "CUDA-graph replays / 10); ms per network evaluation at batch 128 in 'tf32' and 'f16' (median of CUDA-event "
             "timings); per-image rel-L2 of what was timed vs strict fp32",
      gpu=name, power_limit_w=power, clocks=clk, peak_reference=dict(fp16_dense_tflops=PEAK_F16 / 1e12, hbm_tb_s=PEAK_HBM / 1e12),
      attention_block=blocks, ms_per_eval_batch128=speed, rel_l2_vs_fp32_oracle_batch4=error, reps=args.reps,
      networks=NETWORKS,
      config=dict(weights='random init, torch.manual_seed(0); NCSN++ init_scale 1, DDPM zero-init weights re-drawn at scale 1',
                  data='random normal images (x5 for VE), random time labels / log-uniform sigmas in [0.01, 50]'))
  line = json.dumps(rec)
  print(line)
  if args.out:
    with open(args.out, 'w') as fh:
      fh.write(line + '\n')


if __name__ == '__main__':
  main()
