"""`-m gpu`: 3x3 'same' convolutions with 256 output channels on 16- and 32-pixel rows run in the swapped-operand
form (two 128-channel halves of every 256-pixel tile) with the halo mainloop, at every batch size.  Each converted
shape is checked against the strict-fp32 CUDA-core convolution and torch, and the halo mainloop against the
nine-load one (bit-identical: same products in the same K order)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import golden_config, seeded_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


CASES = [
    dict(B=64, H=16, W=16, C1=256, C2=0, Cout=256),     # 128 tiles
    dict(B=3, H=16, W=16, C1=256, C2=0, Cout=256),      # 6 tiles: a batch the row-major plan would cut into 128 columns
    dict(B=64, H=16, W=16, C1=256, C2=256, Cout=256),   # two-source (concat) input, up path
    dict(B=20, H=32, W=32, C1=256, C2=0, Cout=256),     # 32-pixel rows, 160 tiles on 132 persistent CTAs
    dict(B=20, H=32, W=32, C1=256, C2=128, Cout=256),   # 32-pixel rows, two sources (128-channel second source)
]
IDS = lambda c: 'B{B}_{H}x{W}_{C1}+{C2}->{Cout}'.format(**c)


def _operands(case, f16, seed):
  import gpu_util
  B, H, W, C1, C2, Cout = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout'))
  torch.manual_seed(seed)
  cvt = (lambda t: t.half()) if f16 else gpu_util.round_tf32
  x1 = cvt(torch.randn(B, H, W, C1, device='cuda:0'))
  x2 = cvt(torch.randn(B, H, W, C2, device='cuda:0')) if C2 else None
  w = torch.randn(Cout, C1 + C2, 3, 3, device='cuda:0') / np.sqrt((C1 + C2) * 9)
  w = w.half().float() if f16 else gpu_util.round_tf32(w)
  return x1, x2, w


@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_swap_halo256_conv_matches_cuda_core_conv(dev, case, f16):
  """Bias, per-image time-embedding row, residual and scale in the swapped epilogue; fp32 store."""
  import gpu_util
  B, H, W, C1, C2, Cout = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout'))
  if f16 and C2 % 64:
    pytest.skip('fp16 operands need 64-channel chunks')
  x1, x2, w = _operands(case, f16, 36)
  bias = torch.randn(Cout, device=dev)
  rowvec = torch.randn(B, Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  kw = dict(rowvec=rowvec, rowvec_ld=Cout, residual=res, scale=0.7071067690849304)
  wp = gpu_util.pack_conv_weight(w, f16=f16)
  y = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, 3, impl=2 if f16 else 1, **kw)
  x1f, x2f = x1.float(), (x2.float() if x2 is not None else None)
  ref = gpu_util.conv_nhwc(x1f, x2f, gpu_util.pack_conv_weight(w), bias, Cout, 3, impl=0, **kw)
  torch.cuda.synchronize()
  err = (y - ref).abs().max().item()
  assert err < 2e-4 * max(1.0, ref.abs().max().item()), f'max abs err {err}'
  xc = x1f if x2 is None else torch.cat([x1f, x2f], 3)
  tref = (F.conv2d(xc.permute(0, 3, 1, 2), w, bias, padding=1).permute(0, 2, 3, 1) + rowvec[:, None, None, :] + res) * 0.7071067690849304
  assert torch.allclose(y, tref, rtol=2e-4, atol=2e-4), (y - tref).abs().max().item()
  # the TF32-rounded store is exactly the rounding of the plain store
  y2 = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, 3, impl=2 if f16 else 1, round_out=True, **kw)
  assert torch.equal(y2, gpu_util.round_tf32(y))


@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_swap_halo256_equals_nine_load_mainloop(dev, case, f16):
  import gpu_util
  B, H, W, C1, C2, Cout = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'Cout'))
  if f16 and C2 % 64:
    pytest.skip('fp16 operands need 64-channel chunks')
  x1, x2, w = _operands(case, f16, 46)
  wp = gpu_util.pack_conv_weight(w, f16=f16)
  bias = torch.randn(Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  kw = dict(residual=res, scale=0.7071067690849304)
  y_halo = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, 3, impl=2 if f16 else 1, **kw)
  y_nine = gpu_util.conv_nhwc(x1, x2, wp, bias, Cout, 3, impl=5 if f16 else 4, **kw)
  torch.cuda.synchronize()
  assert torch.equal(y_halo, y_nine), (y_halo - y_nine).abs().max().item()


@pytest.mark.parametrize('S2', [0, 256])
def test_swap_halo256_with_fused_skip_projection(dev, S2):
  """(Conv_1(h) + Conv_2(x)) / sqrt(2) at 16x16, 256 -> 256: the extra 1x1 phase of the swapped halo loop."""
  import gpu_util
  B, H, W, C, S1, Cout = 64, 16, 16, 256, 256, 256
  torch.manual_seed(56)
  rt = gpu_util.round_tf32
  x = rt(torch.randn(B, H, W, C, device=dev))
  s1 = rt(torch.randn(B, H, W, S1, device=dev))
  s2 = rt(torch.randn(B, H, W, S2, device=dev)) if S2 else None
  w = rt(torch.randn(Cout, C, 3, 3, device=dev) / np.sqrt(C * 9))
  ws = rt(torch.randn(Cout, S1 + S2, device=dev) / np.sqrt(S1 + S2))
  bias, bias_s = torch.randn(Cout, device=dev), torch.randn(Cout, device=dev)
  sc = 0.7071067690849304
  y = gpu_util.conv_skip_nhwc(x, s1, s2, gpu_util.pack_conv_weight(w), bias, ws.contiguous(), bias_s, Cout, scale=sc)
  torch.cuda.synchronize()
  sx = s1 if s2 is None else torch.cat([s1, s2], 3)
  ref = (F.conv2d(x.permute(0, 3, 1, 2), w, bias, padding=1).permute(0, 2, 3, 1) + sx @ ws.t() + bias_s) * sc
  assert torch.allclose(y, ref, rtol=2e-4, atol=3e-4), (y - ref).abs().max().item()


def test_plan_forms_of_the_headline_network(dev):
  """Every 3x3 'same' convolution with 256 outputs at 16x16 is a swapped halo launch, at batch 1024, at 128 (the
  strong-scaling probe) and at 8 (so that small-batch plans compute each output as the large ones do); the 8x8 and
  4x4 launches keep their row-major tiles."""
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision='f16').to(dev)
  for B in (1024, 128, 8):
    model.engine(B, dev)
    names = model.op_names()
    at16 = [n for n in names if n.startswith('conv3x3') and '->256 @16' in n and ' s2' not in n]
    assert at16 and all('[swap-halo]' in n for n in at16), at16
    low = [n for n in names if n.startswith('conv3x3') and ('@8' in n or '@4' in n)]
    assert low and not any('[swap' in n for n in low), low
  model._release()
