"""`-m gpu`: the wgmma/TMA contraction kernel against the strict-fp32 CUDA-core kernel on
TF32-representable operands (products are then exact in fp32, so only the summation order differs),
then the TF32 execution mode of the whole network and sampler against the strict-fp32 oracle within
the project's 1e-3 per-image relative-L2 tolerance."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3      # the project's parity bound: per-image relative L2 vs reference <= 1e-3


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


CASES = [
    dict(B=2, H=32, W=32, C1=128, C2=0, Cout=128, k=3),
    dict(B=2, H=16, W=16, C1=256, C2=0, Cout=256, k=3),
    dict(B=4, H=8, W=8, C1=256, C2=0, Cout=256, k=3),
    dict(B=3, H=4, W=4, C1=256, C2=0, Cout=256, k=3),      # 48 rows: partial tile, TMA out-of-bounds images
    dict(B=9, H=4, W=4, C1=256, C2=256, Cout=256, k=3),    # two tiles, two-source K loop
    dict(B=2, H=16, W=16, C1=256, C2=128, Cout=256, k=3),  # 384-channel concat
    dict(B=2, H=32, W=32, C1=256, C2=128, Cout=128, k=1),  # 1x1 skip conv
    dict(B=1, H=32, W=32, C1=128, C2=0, Cout=128, k=1),
    dict(B=1, H=64, W=64, C1=32, C2=0, Cout=128, k=3),     # box height 2
    dict(B=1, H=8, W=256, C1=32, C2=0, Cout=128, k=3),     # width > 128: column tiles
    dict(B=40, H=16, W=16, C1=128, C2=0, Cout=256, k=3),   # 80 tiles: fewer than the 132 SMs, one wave
    dict(B=160, H=16, W=16, C1=32, C2=0, Cout=128, k=3),   # 320 tiles on 132 persistent CTAs: several tiles per CTA
    # 3x3 convolutions at both widths that have a halo form (three W-shifted halo copies per channel chunk) in the swapped kernel
    dict(B=2, H=32, W=32, C1=256, C2=128, Cout=128, k=3),  # swapped, two sources, 6 (f16) / 12 (tf32) chunks
    dict(B=4, H=16, W=16, C1=128, C2=0, Cout=128, k=3),    # swapped, 16-pixel rows: one whole image per tile
    dict(B=160, H=16, W=16, C1=256, C2=0, Cout=256, k=3),  # 320 row-major 256-column tiles, multi-wave
    dict(B=20, H=32, W=32, C1=256, C2=128, Cout=256, k=3), # pairs at 32-pixel rows (4 rows per CTA), two sources
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'B{B}_{H}x{W}_{C1}+{C2}->{Cout}_k{k}'.format(**c))
def test_tcgen05_conv_matches_cuda_core_conv(dev, case):
  import gpu_util
  B, H, W, C1, C2, Cout, k = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout', 'k'))
  torch.manual_seed(6)
  rt = gpu_util.round_tf32
  x1 = rt(torch.randn(B, H, W, C1, device=dev))
  x2 = rt(torch.randn(B, H, W, C2, device=dev)) if C2 else None
  w = rt(torch.randn(Cout, C1 + C2, k, k, device=dev) / np.sqrt((C1 + C2) * k * k))
  bias = torch.randn(Cout, device=dev)
  rowvec = torch.randn(B, Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  wp = gpu_util.pack_conv_weight(w)
  kw = dict(rowvec=rowvec, rowvec_ld=Cout, residual=res, scale=0.7071067690849304)
  ref = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=0, **kw)
  y = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=1, **kw)
  torch.cuda.synchronize()
  err = (y - ref).abs().max().item()
  assert err < 2e-4 * max(1.0, ref.abs().max().item()), f'max abs err {err}'
  # and against torch's own fp32 convolution
  xc = x1 if x2 is None else torch.cat([x1, x2], 3)
  tref = (F.conv2d(xc.permute(0, 3, 1, 2), w, bias, padding=k // 2).permute(0, 2, 3, 1) + rowvec[:, None, None, :] + res) * 0.7071067690849304
  assert torch.allclose(y, tref, rtol=2e-4, atol=2e-4)
  # TF32-rounded store is exactly the rounding of the plain store
  y2 = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=1, round_out=True, **kw)
  assert torch.equal(y2, rt(y))


LOWC_CASES = [
    dict(B=2, H=64, W=64, C1=16, C2=0, Cout=16, k=3),      # FFHQ level 0 shape (16 -> 16), 2 x 8 x 2 tiles
    dict(B=1, H=32, W=96, C1=32, C2=0, Cout=32, k=3),
    dict(B=2, H=16, W=32, C1=64, C2=0, Cout=64, k=3),      # four 16-channel slabs
    dict(B=1, H=24, W=64, C1=48, C2=0, Cout=16, k=3),      # concat already materialised (48 channels)
    dict(B=1, H=16, W=64, C1=128, C2=64, Cout=64, k=3),    # 192 channels from two sources
    dict(B=2, H=32, W=32, C1=32, C2=16, Cout=16, k=1),     # two-source 1x1 skip projection
    dict(B=1, H=8, W=32, C1=16, C2=16, Cout=32, k=1),      # a single tile
    dict(B=1, H=40, W=160, C1=16, C2=0, Cout=64, k=3),
]


@pytest.mark.parametrize('case', LOWC_CASES, ids=lambda c: 'B{B}_{H}x{W}_{C1}+{C2}->{Cout}_k{k}'.format(**c))
def test_few_channel_mma_conv_matches_cuda_core_conv(dev, case):
  """conv_lowc.cu (impl 3: warp-level TF32 MMAs, the 16..64-channel levels of the nf=16 networks) against the strict-fp32
  CUDA-core kernel.  On TF32-representable operands the products are exact, so only the summation order differs; on
  arbitrary fp32 operands the kernel rounds them to the TF32 grid itself, i.e. equals impl 0 on pre-rounded operands."""
  import gpu_util
  B, H, W, C1, C2, Cout, k = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout', 'k'))
  torch.manual_seed(11)
  rt = gpu_util.round_tf32
  x1f = torch.randn(B, H, W, C1, device=dev)
  x2f = torch.randn(B, H, W, C2, device=dev) if C2 else None
  wf = torch.randn(Cout, C1 + C2, k, k, device=dev) / np.sqrt((C1 + C2) * k * k)
  x1, x2, w = rt(x1f), (rt(x2f) if C2 else None), rt(wf)
  bias = torch.randn(Cout, device=dev)
  rowvec = torch.randn(B, Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  wp = gpu_util.pack_conv_weight(w)
  kw = dict(rowvec=rowvec, rowvec_ld=Cout, residual=res, scale=0.7071067690849304)
  ref = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=0, **kw)
  y = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=3, **kw)
  torch.cuda.synchronize()
  err = (y - ref).abs().max().item()
  assert err < 2e-5 * max(1.0, ref.abs().max().item()), f'max abs err {err}'
  xc = x1 if x2 is None else torch.cat([x1, x2], 3)
  tref = (F.conv2d(xc.permute(0, 3, 1, 2), w, bias, padding=k // 2).permute(0, 2, 3, 1) + rowvec[:, None, None, :] + res) * 0.7071067690849304
  assert torch.allclose(y, tref, rtol=2e-5, atol=2e-5)
  # unrounded operands: the kernel's own rounding is cvt.rna, the same as round_tf32 -> same result as above, bit for bit
  y_raw = gpu_util.conv_nhwc(x1f, x2f, gpu_util.pack_conv_weight(wf), bias, Cout, k, impl=3, **kw)
  assert torch.equal(y_raw, y)
  # plain epilogue (no bias / row vector / residual) and the TF32-grid store
  y_plain = gpu_util.conv_nhwc(x1, x2, wp, None, Cout, k, impl=3)
  ref_plain = gpu_util.conv_nhwc(x1, x2, wp, None, Cout, k, impl=0)
  assert (y_plain - ref_plain).abs().max().item() < 2e-5 * max(1.0, ref_plain.abs().max().item())
  y2 = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=3, round_out=True, **kw)
  assert torch.equal(y2, rt(y))


def test_few_channel_mma_conv_rejects_other_shapes(dev):
  import gpu_util
  x = torch.randn(1, 8, 32, 24, device=dev)      # 24 channels: not a multiple of 16
  w = gpu_util.pack_conv_weight(torch.randn(16, 24, 3, 3, device=dev))
  with pytest.raises(RuntimeError, match='conv_lowc'):
    gpu_util.conv_nhwc(x, None, w, None, 16, 3, impl=3)
  x = torch.randn(1, 8, 16, 16, device=dev)      # 16 pixels wide: no 32-pixel tile
  w = gpu_util.pack_conv_weight(torch.randn(16, 16, 3, 3, device=dev))
  with pytest.raises(RuntimeError, match='conv_lowc'):
    gpu_util.conv_nhwc(x, None, w, None, 16, 3, impl=3)


F16_CASES = [c for c in CASES if c['C1'] % 64 == 0 and c['C2'] % 64 == 0]


@pytest.mark.parametrize('case', F16_CASES, ids=lambda c: 'B{B}_{H}x{W}_{C1}+{C2}->{Cout}_k{k}'.format(**c))
def test_tcgen05_f16_conv_matches_torch(dev, case):
  """kind::f16 form of the same contraction: activations and packed weights are IEEE fp16 in memory (64-channel
  K steps), accumulation and epilogue are fp32.  fp16 x fp16 products are exact in fp32, so against torch's fp32
  convolution of the SAME fp16-representable values only the summation order differs."""
  import gpu_util
  B, H, W, C1, C2, Cout, k = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout', 'k'))
  torch.manual_seed(6)
  x1 = torch.randn(B, H, W, C1, device=dev).half()
  x2 = torch.randn(B, H, W, C2, device=dev).half() if C2 else None
  w = (torch.randn(Cout, C1 + C2, k, k, device=dev) / np.sqrt((C1 + C2) * k * k)).half().float()
  bias = torch.randn(Cout, device=dev)
  rowvec = torch.randn(B, Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  wp = gpu_util.pack_conv_weight(w, f16=True)
  assert torch.equal(wp.float().reshape(k * k, Cout, C1 + C2), w.permute(2, 3, 0, 1).reshape(k * k, Cout, C1 + C2))
  kw = dict(rowvec=rowvec, rowvec_ld=Cout, residual=res, scale=0.7071067690849304)
  y = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=2, **kw)
  torch.cuda.synchronize()
  xc = x1.float() if x2 is None else torch.cat([x1.float(), x2.float()], 3)
  tref = (F.conv2d(xc.permute(0, 3, 1, 2), w, bias, padding=k // 2).permute(0, 2, 3, 1) + rowvec[:, None, None, :] + res) * 0.7071067690849304
  assert torch.allclose(y, tref, rtol=2e-4, atol=2e-4), (y - tref).abs().max().item()


HALO_CASES = [c for c in CASES if c['k'] == 3 and c['W'] in (16, 32) and (c['Cout'] == 128 or c['B'] * c['H'] * c['W'] >= 132 * 128)]


@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('case', HALO_CASES, ids=lambda c: 'B{B}_{H}x{W}_{C1}+{C2}->{Cout}_k{k}'.format(**c))
def test_halo_mainloop_equals_nine_load_mainloop(dev, case, f16):
  """impl 1 / 2: halo form in the swapped kernel (the default plan), 4 / 5: one shifted tile load per filter tap
  everywhere.  Same operands, same products: the nine-load loop of a shape that has a halo form walks K in the halo
  form's order (channel chunk, filter column, filter row), so on / off are bit-identical.  What differs in mechanism:
  zero fill of a shifted tile vs of a halo copy at the borders, and the operand addressing."""
  import gpu_util
  B, H, W, C1, C2, Cout, k = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout', 'k'))
  if f16 and (C1 % 64 or C2 % 64):
    pytest.skip('fp16 operands need 64-channel chunks')
  torch.manual_seed(26)
  cvt = (lambda t: t.half()) if f16 else gpu_util.round_tf32
  x1 = cvt(torch.randn(B, H, W, C1, device=dev))
  x2 = cvt(torch.randn(B, H, W, C2, device=dev)) if C2 else None
  w = torch.randn(Cout, C1 + C2, k, k, device=dev) / np.sqrt((C1 + C2) * k * k)
  w = w.half().float() if f16 else gpu_util.round_tf32(w)
  wp = gpu_util.pack_conv_weight(w, f16=True) if f16 else gpu_util.pack_conv_weight(w)
  bias = torch.randn(Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  kw = dict(residual=res, scale=0.7071067690849304)
  y_default = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=2 if f16 else 1, **kw)
  y_nine = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, k, impl=5 if f16 else 4, **kw)
  torch.cuda.synchronize()
  e1 = (y_default - y_nine).abs().max().item()
  print(f'halo vs nine-load mainloop {"f16" if f16 else "tf32"} B{B} {H}x{W} {C1}+{C2}->{Cout}: max abs diff {e1:.2e}')
  assert torch.equal(y_default, y_nine)


SKIP_CASES = [
    dict(B=2, H=16, W=16, C=256, S1=256, S2=256, Cout=256),     # up-path block: concat skip input, single-CTA tiles
    dict(B=160, H=16, W=16, C=256, S1=256, S2=128, Cout=256),   # multi-wave row-major 256-column tiles
    dict(B=2, H=32, W=32, C=128, S1=256, S2=128, Cout=128),     # swapped-operand form (128 output channels)
    dict(B=3, H=4, W=4, C=256, S1=256, S2=0, Cout=256),         # partial tile
    dict(B=4, H=8, W=8, C=256, S1=128, S2=0, Cout=256),         # level change 128 -> 256
]


@pytest.mark.parametrize('case', SKIP_CASES, ids=lambda c: 'B{B}_{H}x{W}_{C}|{S1}+{S2}->{Cout}'.format(**c))
def test_tcgen05_conv_with_fused_skip_projection(dev, case):
  """Resblock tail (layerspp.py:268-274): (Conv_1(h) + Conv_2(x)) / sqrt(2) as ONE contraction whose K loop
  appends the 1x1 projection of the (two-source) block input to the nine taps of the 3x3 filter."""
  import gpu_util
  B, H, W, C, S1, S2, Cout = (case[x] for x in ('B', 'H', 'W', 'C', 'S1', 'S2', 'Cout'))
  torch.manual_seed(16)
  rt = gpu_util.round_tf32
  x = rt(torch.randn(B, H, W, C, device=dev))
  s1 = rt(torch.randn(B, H, W, S1, device=dev))
  s2 = rt(torch.randn(B, H, W, S2, device=dev)) if S2 else None
  w = rt(torch.randn(Cout, C, 3, 3, device=dev) / np.sqrt(C * 9))
  ws = rt(torch.randn(Cout, S1 + S2, device=dev) / np.sqrt(S1 + S2))
  bias, bias_s = torch.randn(Cout, device=dev), torch.randn(Cout, device=dev)
  wp = gpu_util.pack_conv_weight(w)
  sc = 0.7071067690849304
  y = gpu_util.conv_skip_nhwc(x, s1, s2, wp, bias, ws.contiguous(), bias_s, Cout, scale=sc)
  torch.cuda.synchronize()
  sx = s1 if s2 is None else torch.cat([s1, s2], 3)
  ref = (F.conv2d(x.permute(0, 3, 1, 2), w, bias, padding=1).permute(0, 2, 3, 1) + sx @ ws.t() + bias_s) * sc
  assert torch.allclose(y, ref, rtol=2e-4, atol=3e-4), (y - ref).abs().max().item()
  # equals the unfused pair of launches (1x1 projection, then 3x3 with a residual) up to summation order
  wsp = gpu_util.pack_conv_weight(ws.reshape(Cout, S1 + S2, 1, 1))
  s = gpu_util.conv_nhwc(s1, s2, wsp, bias_s, Cout, 1, impl=1)
  y2 = gpu_util.conv_nhwc(x, None, wp, bias, Cout, 3, residual=s, scale=sc, impl=1)
  assert torch.allclose(y, y2, rtol=1e-5, atol=2e-5), (y - y2).abs().max().item()


@pytest.mark.parametrize('nimg', [1, 3, 200])
def test_fused_attention_core_matches_torch(dev, nimg):
  """layerspp.py:82-91 in one kernel: softmax(q k^T / sqrt(C)) v + b_v, NIN_3, (x + h)/sqrt(2), and the quad sums of
  the result.  nimg=200 -> 400 tiles on 132 persistent CTAs (ring reuse across tiles, odd tile counts)."""
  import gpu_util
  rt = gpu_util.round_tf32
  torch.manual_seed(21 + nimg)
  T = C = 256
  q = rt(torch.randn(nimg, T, C, device=dev) * 1.5)
  k = rt(torch.randn(nimg, T, C, device=dev) * 1.5)
  v = rt(torch.randn(nimg, T, C, device=dev))
  w3 = rt(torch.randn(C, C, device=dev) / 16)           # [out][in]
  bv, b3 = torch.randn(C, device=dev), torch.randn(C, device=dev)
  x = torch.randn(nimg * T, C, device=dev)
  qk = torch.cat([q, k], 2).reshape(nimg * T, 2 * C).contiguous()
  vT = v.transpose(1, 2).contiguous()
  sc = 0.7071067690849304
  out, qs = gpu_util.attention_core(qk, vT, w3, bv, b3, x, sc, want_stats=True)
  torch.cuda.synchronize()
  P = torch.softmax(torch.bmm(q, k.transpose(1, 2)) * (C ** -0.5), dim=-1)
  h = torch.bmm(P, v) + bv
  ref = ((h.reshape(nimg * T, C) @ w3.t() + b3) + x) * sc
  err = ((out - ref).norm() / ref.norm()).item()
  assert err < 3e-4, err                                  # TF32 operands (E, O') inside the chain
  assert (out - ref).abs().max().item() < 5e-3
  # quad sums of what was stored
  o4 = out.reshape(nimg, T, C // 4, 4).double()
  assert torch.allclose(qs[..., 0], o4.sum((1, 3)), rtol=1e-5, atol=1e-3)
  assert torch.allclose(qs[..., 1], (o4 * o4).sum((1, 3)), rtol=1e-5, atol=1e-3)
  # peaked softmax rows (large logits): the max subtraction must keep exp() in range
  qk2 = (qk * 6).contiguous()
  out2 = gpu_util.attention_core(rt(qk2), vT, w3, bv, b3, x, sc)
  P2 = torch.softmax(torch.bmm(rt(q * 6), rt(k * 6).transpose(1, 2)) * (C ** -0.5), dim=-1)
  ref2 = (((torch.bmm(P2, v) + bv).reshape(nimg * T, C) @ w3.t() + b3) + x) * sc
  assert torch.isfinite(out2).all()
  assert ((out2 - ref2).norm() / ref2.norm()).item() < 3e-4


@pytest.mark.parametrize('nimg', [2, 150])
def test_fused_attention_core_f16_matches_torch(dev, nimg):
  """The kind::f16 variant (fp16 q|k, v^T, W3 in memory; E and O' staged as fp16; 3-stage ring)."""
  import gpu_util
  torch.manual_seed(31 + nimg)
  T = C = 256
  q = (torch.randn(nimg, T, C, device=dev) * 1.5).half()
  k = (torch.randn(nimg, T, C, device=dev) * 1.5).half()
  v = torch.randn(nimg, T, C, device=dev).half()
  w3 = (torch.randn(C, C, device=dev) / 16).half()
  bv, b3 = torch.randn(C, device=dev), torch.randn(C, device=dev)
  x = torch.randn(nimg * T, C, device=dev)
  qk = torch.cat([q, k], 2).reshape(nimg * T, 2 * C).contiguous()
  vT = v.transpose(1, 2).contiguous()
  sc = 0.7071067690849304
  out, qs = gpu_util.attention_core(qk, vT, w3, bv, b3, x, sc, want_stats=True)
  torch.cuda.synchronize()
  P = torch.softmax(torch.bmm(q.float(), k.float().transpose(1, 2)) * (C ** -0.5), dim=-1)
  h = torch.bmm(P, v.float()) + bv
  ref = ((h.reshape(nimg * T, C) @ w3.float().t() + b3) + x) * sc
  err = ((out - ref).norm() / ref.norm()).item()
  assert err < 3e-4, err
  o4 = out.reshape(nimg, T, C // 4, 4).double()
  assert torch.allclose(qs[..., 0], o4.sum((1, 3)), rtol=1e-5, atol=1e-3)


def test_tcgen05_batched_gemm_attention_shapes(dev):
  import gpu_util
  rt = gpu_util.round_tf32
  torch.manual_seed(7)
  nb, T, C = 3, 256, 256
  qk = rt(torch.randn(nb * T, 2 * C, device=dev) * 0.3)
  # S[b] = q[b] k[b]^T with q,k interleaved in one [B*T, 2C] buffer (pitch 2C)
  S = gpu_util.gemm_nt(qk, qk[:, C:], nb, T, T, C, lda=2 * C, ldw=2 * C, impl=1)
  ref = torch.bmm(qk[:, :C].reshape(nb, T, C), qk[:, C:].reshape(nb, T, C).transpose(1, 2)).reshape(nb * T, T)
  assert torch.allclose(S, ref, rtol=2e-4, atol=2e-3)
  # v^T[b] = Wv a[b]^T : shared row operand, batched column operand
  Wv = rt(torch.randn(C, C, device=dev) / 16)
  a = rt(torch.randn(nb * T, C, device=dev))
  vT = gpu_util.gemm_nt(Wv, a, nb, C, T, C, a_batch_rows=0, w_batch_rows=T, impl=1)
  refv = torch.einsum('ci,bti->bct', Wv, a.view(nb, T, C)).reshape(nb * C, T)
  assert torch.allclose(vT, refv, rtol=2e-4, atol=2e-3)
  # projection with N = 2C = 512 (two N tiles) and a bias
  Wqk = rt(torch.randn(2 * C, C, device=dev) / 16)
  b = torch.randn(2 * C, device=dev)
  out = gpu_util.gemm_nt(a, Wqk, 1, nb * T, 2 * C, C, w_batch_rows=0, bias=b, impl=1)
  assert torch.allclose(out, a @ Wqk.t() + b, rtol=2e-4, atol=2e-3)


@pytest.mark.parametrize('precision', ['tf32', 'f16'])
def test_forward_tf32_cifar10_matches_oracle_within_parity_bound(dev, precision):
  """Both tensor-core operand formats (TF32-rounded fp32, fp16: 11-bit significands either way) against the
  strict-fp32 oracle and the reference's own CPU output, same bound."""
  g = golden('ncsnpp_cifar10_ve.npz')
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision=precision, keep_activations=True).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  x, sigma = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma, taps=taps)
    y = model(x, sigma)
  rows = []
  for i in sorted(taps):
    try:
      rows.append((i, rel_l2(model.tap(i), taps[i])))
    except RuntimeError:
      pass
  worst = sorted(rows, key=lambda r: -r[1])[:5]
  assert all(r[1] < 5e-3 for r in rows), f'worst modules (index, rel-L2): {worst}'
  e_or, e_gold = rel_l2(y, ref), rel_l2(y, torch.from_numpy(g['y']).to(dev))
  print(f'cifar10 {precision} single-eval rel-L2 vs GPU oracle {e_or:.3e}, vs reference CPU golden {e_gold:.3e}; worst taps {worst}')
  assert e_or < TOL_PARITY and e_gold < TOL_PARITY


def test_forward_fp32_cifar10_matches_oracle(dev):
  g = golden('ncsnpp_cifar10_ve.npz')
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision='fp32').to(dev)
  x, sigma = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  y = model(x, sigma)
  assert rel_l2(y, torch.from_numpy(g['y']).to(dev)) < 1e-4


@pytest.mark.parametrize('precision', ['tf32', 'f16'])
def test_pc_sampler_tf32_cifar10_K_steps_within_parity_bound(dev, precision):
  """K PC iterations (2K network evaluations) of the headline sampler at B=8 vs the strict-fp32 oracle."""
  from score_sde_pytorch_b200 import sampling, sde_lib, native
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (8, 3, 32, 32)
  K = 10
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  torch.manual_seed(1)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(1)
  ref, _ = SO.pc_sample(osde, lambda x, l: NO.ncsnpp_forward(sd, cfg, x, l), shape, eps=1e-5, device=dev,
                        x_init=x0, num_iters=K)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor,
                              corrector=sampling.LangevinCorrector, shape=shape, snr=0.16, n_steps=1,
                              probability_flow=False, continuous=True, eps=1e-5, device=dev)
  torch.cuda.manual_seed(1)
  x, x_mean = plan.run(x0, first_step=0, num_steps=K)
  e = rel_l2(x_mean, ref)
  print(f'cifar10 {precision} {K}-step PC rel-L2 vs oracle: {e:.3e}')
  assert e < TOL_PARITY


@pytest.mark.parametrize('precision', ['f16', 'tf32'])
def test_pc_sampler_cifar10_full_1000_steps_within_parity_bound(dev, precision):
  """The north-star statement itself: the COMPLETE 1000-step VE predictor-corrector sampler (2000 network
  evaluations, same prior draw and same CUDA noise stream) against the strict-fp32 oracle loop, per-image
  relative L2 <= 1e-3.  Batch 4 keeps the oracle to about a minute."""
  from score_sde_pytorch_b200 import sampling, sde_lib, native
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (4, 3, 32, 32)
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  torch.manual_seed(11)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(11)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, lambda x, l: NO.ncsnpp_forward(sd, cfg, x, l), shape, eps=1e-5, device=dev, x_init=x0)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor,
                              corrector=sampling.LangevinCorrector, shape=shape, snr=0.16, n_steps=1,
                              probability_flow=False, continuous=True, eps=1e-5, device=dev)
  torch.cuda.manual_seed(11)
  x, x_mean = plan.run(x0, first_step=0, num_steps=1000)
  e = rel_l2(x_mean, ref)
  print(f'cifar10 {precision} full 1000-step PC sampler rel-L2 vs oracle: {e:.3e}')
  assert torch.isfinite(x_mean).all()
  assert e < TOL_PARITY
