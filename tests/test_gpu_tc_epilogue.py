"""`-m gpu`: the tensor-core contraction's epilogue writes through shared memory and TMA stores, which clip at the
output tensor map's bounds.  Every value must match a float64 reference, and nothing outside the output window may
be written: a sentinel in the pitch padding (an output pitch wider than N) and in the rows past M must survive.
Covers row-major tiles (128 and 256 columns) and swapped tiles, with and without the TMA-loaded residual, for fp32,
TF32-rounded and fp16 stores, with TF32 and fp16 operands."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from score_sde_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
SENTINEL = -12345.0
EXTRA_ROWS = 7


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _tol(mode):
  # fp32 stores: summation order only; TF32 / fp16 stores add one rounding of the stored value (2^-11 relative)
  return dict(rtol=2e-4, atol=2e-4) if mode == 0 else dict(rtol=1.2e-3, atol=1e-3)


def _operands(shape, f16, dev, scale=1.0):
  import gpu_util
  x = torch.randn(*shape, device=dev) * scale
  return x.half() if f16 else gpu_util.round_tf32(x)


# (m, n, k): single-batch GEMMs whose M is not a multiple of 128; n = 128 -> 128-column row-major tiles, n = 256 with
# more than half an SM wave of row tiles -> 256-column tiles
GEMM_CASES = [(200, 128, 64), (9010, 256, 128), (77, 256, 64)]


@pytest.mark.parametrize('mode', [0, 1, 2], ids=['fp32', 'tf32', 'fp16'])
@pytest.mark.parametrize('f16', [False, True], ids=['tf32ops', 'f16ops'])
@pytest.mark.parametrize('mnk', GEMM_CASES, ids=lambda c: 'm{}_n{}_k{}'.format(*c))
def test_gemm_epilogue_stays_inside_output_window(dev, mnk, f16, mode):
  m, n, k = mnk
  torch.manual_seed(11)
  a = _operands((m, k), f16, dev)
  w = _operands((n, k), f16, dev, 1 / np.sqrt(k))
  bias = torch.randn(n, device=dev)
  ldo = n + 24                               # pitch padding of 24 elements (a multiple of 8: fp16 rows stay 16-byte aligned)
  out = torch.full((m + EXTRA_ROWS, ldo), SENTINEL, device=dev, dtype=torch.float16 if mode == 2 else torch.float32)
  _lib.call('b200_gemm_nt_f32', _lib.ptr(a), k, m, _lib.ptr(w), k, n, 1, m, n, k, _lib.ptr(bias), mode, _lib.ptr(out),
            ldo, 2 if f16 else 1, _lib.stream_ptr(dev))
  torch.cuda.synchronize()
  ref = a.double() @ w.double().t() + bias.double()
  y = out[:m, :n].double()
  assert torch.allclose(y, ref, **_tol(mode)), (y - ref).abs().max().item()
  assert bool((out[:m, n:] == SENTINEL).all()), 'pitch padding written'
  assert bool((out[m:] == SENTINEL).all()), 'rows past M written'


# swapped form (128 output channels; 3x3 on 32- / 16-pixel rows: halo mainloop; 1x1) and row-major tiles
CONV_CASES = [
    dict(B=2, H=32, W=32, C=128, Cout=128, k=3),
    dict(B=4, H=16, W=16, C=128, Cout=256, k=3),
    dict(B=2, H=32, W=32, C=128, Cout=128, k=1),
    dict(B=160, H=8, W=8, C=128, Cout=256, k=3),
    dict(B=9, H=4, W=4, C=256, Cout=256, k=3),     # row-major, M = 144: a tail tile whose residual rows past M are zero-filled
]


@pytest.mark.parametrize('mode', [0, 1, 2], ids=['fp32', 'tf32', 'fp16'])
@pytest.mark.parametrize('f16', [False, True], ids=['tf32ops', 'f16ops'])
@pytest.mark.parametrize('case', CONV_CASES, ids=lambda c: 'B{B}_{H}x{W}_{C}->{Cout}_k{k}'.format(**c))
def test_conv_residual_epilogue_stays_inside_output_window(dev, case, f16, mode):
  import gpu_util
  B, H, W, C, Cout, k = (case[x] for x in ('B', 'H', 'W', 'C', 'Cout', 'k'))
  torch.manual_seed(12)
  x = _operands((B, H, W, C), f16, dev)
  wt = _operands((Cout, C, k, k), f16, dev, 1 / np.sqrt(C * k * k)).float()
  wp = gpu_util.pack_conv_weight(wt, f16=f16)
  bias = torch.randn(Cout, device=dev)
  rowvec = torch.randn(B, Cout, device=dev)
  res = torch.randn(B, H, W, Cout, device=dev)
  scale = 0.7071067690849304
  M = B * H * W
  out = torch.full((M + EXTRA_ROWS, Cout), SENTINEL, device=dev, dtype=torch.float16 if mode == 2 else torch.float32)
  _lib.call('b200_conv_nhwc_f32', _lib.ptr(x), C, None, 0, B, H, W, _lib.ptr(wp), _lib.ptr(bias), Cout, k,
            _lib.ptr(rowvec), Cout, _lib.ptr(res), scale, mode, _lib.ptr(out), 2 if f16 else 1, _lib.stream_ptr(dev))
  torch.cuda.synchronize()
  conv = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), bias.double(), padding=k // 2).permute(0, 2, 3, 1)
  ref = ((conv + rowvec.double()[:, None, None, :] + res.double()) * scale).reshape(M, Cout)
  y = out[:M].double()
  assert torch.allclose(y, ref, **_tol(mode)), (y - ref).abs().max().item()
  assert bool((out[M:] == SENTINEL).all()), 'rows past M written'
