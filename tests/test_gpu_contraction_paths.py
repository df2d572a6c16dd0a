"""`-m gpu`: the contraction paths only the engine reaches, each against a float64 reference of the same operation on the
operands exactly as the kernel reads them.

  a. the tensor-core contraction's fused GroupNorm quad sums and per-image row vectors (every orientation, store format
     and residual variant of the staged epilogue; images of 16 and 64 rows inside one 128-row tile; the M tail);
  b. the two network heads: the tensor-core NCHW head ((acc + bias) / sigma, n_valid channels of a padded 128-row
     weight tile) and the CUDA-core conv3x3_small_n;
  c. stride-2 VALID convolutions (DDPM's Downsample with_conv: F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 conv);
  d. split TF32 (3xTF32) on every mainloop form;
  e. the few-channel convolution with GroupNorm+SiLU applied on load, and its output quad sums.

Operands are on the TF32 grid or fp16, so every product is exact in fp32 and only the accumulation differs from the
float64 reference.  Per element the bound is K 2^-23 (|x| * |w|)[i] + 1e-6, where |x| * |w| is the same contraction of
absolute values (plus the absolute epilogue terms) and K the number of fp32 additions behind an output; a TF32 / fp16
store adds 2^-11 |ref|.  It is a worst case, not a tuned tolerance: a wrong tap, K chunk or image is off by orders of
magnitude.  Where the code promises bit equality (store formats of one plan, GroupNorm on load) the test asserts it.
Every output buffer is filled with a sentinel that must survive past the output; every quad-sum buffer is zero inside
its [img][N/4][2] window and a sentinel past it.  Each check prints its largest error as a fraction of its bound."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from score_sde_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu
U = 2.0 ** -23
SENT = -12345.0          # output sentinel
QSENT = 7777.0           # quad-sum sentinel
SLACK = 4096             # sentinel elements past every output
STATS_REL = 2e-5         # fp32 partial sums of up to 256 values, added in fp64


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _gen(dev, seed):
  return torch.Generator(device=dev).manual_seed(seed)


def _tc(dev, **fields):
  import gpu_util
  return gpu_util.tc_contract(dev, **fields)


def _out(numel, mode, dev):
  return torch.full((numel + SLACK,), SENT, device=dev, dtype=torch.float16 if mode == 2 else torch.float32)


def _qbuf(nimg, n, dev):
  q = torch.full((nimg * (n // 4) * 2 + 64,), QSENT, device=dev, dtype=torch.float64)
  q[:nimg * (n // 4) * 2] = 0
  return q


def _check_bound(what, y, ref, absref, K, mode):
  """|y - ref| <= K 2^-23 absref + 1e-6, plus one rounding of the stored value for TF32 / fp16 stores."""
  bound = K * U * absref + 1e-6
  if mode:
    bound = bound * (1 + 2.0 ** -11) + 2.0 ** -11 * ref.abs()
  r = ((y.double() - ref).abs() / bound).max().item()
  print(f'[bound] {what}: max |err| / bound = {r:.3e}')
  assert r <= 1.0, f'{what}: error {r:.3g}x its bound'


def _check_sentinel(buf, n, what):
  assert bool((buf[n:] == SENT).all()), f'{what}: written past the output'


def _check_stats(what, q, y, img, nimg, n):
  """q: the kernel's quad sums [img][n/4][2] (+ sentinels); y [rows, n]: the stored values, img [rows] their images."""
  w = nimg * (n // 4) * 2
  assert bool((q[w:] == QSENT).all()), f'{what}: quad sums written past their window'
  q = q[:w].view(nimg, n // 4, 2)
  yq = y.double().view(-1, n // 4, 4)
  z = torch.zeros(nimg, n // 4, device=y.device, dtype=torch.float64)
  s = z.index_add(0, img, yq.sum(2))
  s2 = z.index_add(0, img, (yq * yq).sum(2))
  sa = z.index_add(0, img, yq.abs().sum(2))
  r1 = ((q[..., 0] - s).abs() / (STATS_REL * sa + 1e-30)).max().item()
  r2 = ((q[..., 1] - s2).abs() / (STATS_REL * s2 + 1e-30)).max().item()
  print(f'[stats] {what}: max |d sum| / bound = {r1:.3e}, max |d sumsq| / bound = {r2:.3e}')
  assert r1 <= 1.0 and r2 <= 1.0, f'{what}: quad sums off by {max(r1, r2):.3g}x their bound'
  return sa


def _conv64(x, w, stride=1, valid_pad=False):
  """NHWC x (float64), OIHW w -> NHWC: 'same' padding, or F.pad(x, (0, 1, 0, 1)) + VALID for stride 2."""
  xn = x.permute(0, 3, 1, 2)
  k = w.shape[-1]
  if valid_pad:
    y = F.conv2d(F.pad(xn, (0, 1, 0, 1)), w, stride=stride)
  else:
    y = F.conv2d(xn, w, stride=stride, padding=k // 2)
  return y.permute(0, 2, 3, 1)


def _grid(t, f16):
  """t (fp32) as the kernel's operand: fp16 elements, or fp32 on the TF32 grid; and the float64 of those values."""
  import gpu_util
  op = t.half() if f16 else gpu_util.round_tf32(t)
  return op, op.double()


# ---------------------------------------------------------------------------------------------------------------------
# a. fused GroupNorm quad sums and per-image row vectors
# ---------------------------------------------------------------------------------------------------------------------
# Integer operands in {-1, 0, 1}: every partial sum is exact, so the stored value is exactly acc + the epilogue terms.  The
# bias carries a fractional 1/32 and outputs sit around 200, where the TF32 grid spacing is 1/8 or coarser: every mode-1
# store rounds each value down by exactly 1/32 (|v| >= 128), so quad sums taken before that rounding are off by
# sum(v) / (32 |v|) ~ 1.6e-4 of sum |v|, eight times the bound - random data would average that bias away.
def _int_operand(shape, gen, dev):
  return torch.randint(-1, 2, shape, device=dev, generator=gen).float()


def _epilogue_terms(gen, nrow, n, dev):
  bias = 200 + torch.randint(-20, 21, (n,), device=dev, generator=gen).float() + 1 / 32
  rowvec = torch.randint(-20, 21, (nrow, n), device=dev, generator=gen).float()
  return bias, rowvec


def _run_modes(dev, what, fields, ref, absref, K, rows, n, ld_out, img, nimg, form):
  """Launch the same contraction in store modes 0, 1, 2 with quad sums; check forms, bounds, sentinels, stats, and the
  bit-exact relations between the three store formats."""
  ys, qs = {}, {}
  for mode in (0, 1, 2):
    out = _out(rows * ld_out, mode, dev)
    q = _qbuf(nimg, n, dev)
    got = _tc(dev, out=out, ld_out=ld_out, store_mode=mode, qstats=q, **fields)
    torch.cuda.synchronize()
    assert got == form, f'{what}: form {got!r}, expected {form!r}'
    _check_sentinel(out, rows * ld_out, what)
    y = out[:rows * ld_out].view(rows, ld_out)[:, :n]
    _check_bound(f'{what} mode {mode}', y, ref, absref, K, mode)
    ys[mode], qs[mode] = y, q
    if mode < 2:
      sa = _check_stats(f'{what} mode {mode}', q, y, img, nimg, n)
  import gpu_util
  assert torch.equal(ys[1], gpu_util.round_tf32(ys[0].contiguous())), f'{what}: mode 1 != round_tf32(mode 0)'
  assert torch.equal(ys[2], ys[0].half()), f'{what}: mode 2 != (mode 0).half()'
  w = nimg * (n // 4) * 2
  # mode 2 sums the same fp32 values as mode 0; the fp64 atomics add them in another order
  d = (qs[2][:w] - qs[0][:w]).view(nimg, n // 4, 2).abs()
  assert bool((d[..., 0] <= 1e-12 * sa).all()) and bool((d[..., 1] <= 1e-12 * qs[0][:w].view(nimg, n // 4, 2)[..., 1]).all()), \
      f'{what}: mode-2 quad sums differ from mode 0'
  assert bool((qs[2][w:] == QSENT).all()), f'{what}: mode-2 quad sums written past their window'


STATS_CONV = [
    dict(B=2, H=32, W=32, C=128, N=128, k=3, form='swap-halo'),
    dict(B=4, H=16, W=16, C=256, N=256, k=3, form='swap-halo'),     # two 128-channel halves per tile
    dict(B=2, H=32, W=32, C=256, N=128, k=1, form='swap'),
    dict(B=2, H=8, W=256, C=128, N=128, k=3, form='swap'),          # rows wider than 128 pixels: no halo form
    dict(B=320, H=8, W=8, C=128, N=256, k=3, form='single256'),     # 64-row images, 160 tiles: persistent CTAs
    dict(B=9, H=4, W=4, C=256, N=256, k=3, form='single128'),       # 16-row images, M tail at 144 rows
    dict(B=1, H=64, W=64, C=128, N=256, k=3, form='single128'),     # 64-pixel rows
]


def _stats_conv(dev, case, f16, res, rowvec_ld, seed):
  B, H, W, C, N, k = (case[x] for x in ('B', 'H', 'W', 'C', 'N', 'k'))
  g = _gen(dev, seed)
  x = _int_operand((B, H, W, C), g, dev)
  wt = _int_operand((N, C, k, k), g, dev)
  bias, rowvec = _epilogue_terms(g, B if rowvec_ld else 1, N, dev)
  M, HW = B * H * W, H * W
  resid = torch.randint(-20, 21, (M, N), device=dev, generator=g).float() if res else None
  import gpu_util
  xo = x.half() if f16 else x
  wp = gpu_util.pack_conv_weight(wt, f16=f16)
  img = torch.arange(M, device=dev) // HW
  rv = rowvec.double()[img] if rowvec_ld else rowvec.double()[0].expand(M, N)
  ref = _conv64(x.double(), wt.double(), 1).reshape(M, N) + bias.double() + rv
  absref = _conv64(x.double().abs(), wt.double().abs(), 1).reshape(M, N) + bias.double().abs() + rv.abs()
  if res:
    ref, absref = ref + resid.double(), absref + resid.double().abs()
  fields = dict(a1=xo, c1=C, conv=1, h=H, w=W, nimg=B, taps=k * k, f16=int(f16), wt=wp, n_total=N, k_total=C,
                w_rows=k * k * N, nbatch=1, bias=bias, rowvec=rowvec, rowvec_ld=rowvec_ld, residual=resid,
                ld_res=N if res else 0, rows_per_img=HW)
  what = 'B{B} {H}x{W} {C}->{N} k{k}'.format(**case) + (' f16' if f16 else ' tf32') + (' +res' if res else '') + \
         ('' if rowvec_ld else ' rowvec_ld=0')
  _run_modes(dev, what, fields, ref, absref, C * k * k + 4, M, N, N, img, B, case['form'])


@pytest.mark.parametrize('res', [False, True], ids=['nores', 'res'])
@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('case', STATS_CONV, ids=lambda c: 'B{B}_{H}x{W}_{C}-{N}_k{k}'.format(**c))
def test_conv_quad_sums_and_rowvec(dev, case, f16, res):
  _stats_conv(dev, case, f16, res, case['N'], 21)


@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('case', [STATS_CONV[0], STATS_CONV[5]], ids=['swap', 'rowmajor'])
def test_conv_image_independent_rowvec(dev, case, f16):
  """rowvec_ld = 0: one row vector for every image (uniform labels; the fused skip projection's bias)."""
  _stats_conv(dev, case, f16, True, 0, 22)


# batched GEMMs as the attention projections issue them: (nbatch, M per batch, N, K, A pitch, rows between A batches,
# W pitch, rows between W batches, rows per image); residual pitch N + 16
STATS_GEMM = [
    dict(nb=1, M=1000, N=256, K=128, lda=128, abr=0, ldw=128, wbr=0, T=256),      # M tail inside a 16-row warp block
    dict(nb=1, M=1000, N=256, K=128, lda=128, abr=0, ldw=128, wbr=0, T=64),
    dict(nb=1, M=1000, N=128, K=128, lda=128, abr=0, ldw=128, wbr=0, T=16),
    dict(nb=2, M=256, N=128, K=192, lda=256, abr=256, ldw=192, wbr=0, T=64),      # shared W, A pitch > K
    dict(nb=3, M=128, N=256, K=128, lda=128, abr=0, ldw=160, wbr=256, T=16),      # shared A, W pitch > K
]


@pytest.mark.parametrize('res', [False, True], ids=['nores', 'res'])
@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('case', STATS_GEMM, ids=lambda c: 'nb{nb}_M{M}_N{N}_K{K}_T{T}_abr{abr}_wbr{wbr}'.format(**c))
def test_gemm_quad_sums_and_rowvec(dev, case, f16, res):
  nb, M, N, K, lda, abr, ldw, wbr, T = (case[x] for x in ('nb', 'M', 'N', 'K', 'lda', 'abr', 'ldw', 'wbr', 'T'))
  g = _gen(dev, 23)
  a_rows = abr * (nb - 1) + M if abr else M
  w_rows = wbr * (nb - 1) + N if wbr else N
  A = _int_operand((a_rows, lda), g, dev)
  Wm = _int_operand((w_rows, ldw), g, dev)
  rows = nb * M
  nimg = (rows + T - 1) // T
  bias, rowvec = _epilogue_terms(g, nimg, N, dev)
  ldr = N + 16
  resid = torch.randint(-20, 21, (rows, ldr), device=dev, generator=g).float() if res else None
  img = torch.arange(rows, device=dev) // T
  A64, W64 = A.double(), Wm.double()
  ref = torch.cat([A64[b * abr:b * abr + M, :K] @ W64[b * wbr:b * wbr + N, :K].t() for b in range(nb)])
  absref = torch.cat([A64[b * abr:b * abr + M, :K].abs() @ W64[b * wbr:b * wbr + N, :K].abs().t() for b in range(nb)])
  ref = ref + bias.double() + rowvec.double()[img]
  absref = absref + bias.double().abs() + rowvec.double()[img].abs()
  if res:
    ref, absref = ref + resid.double()[:, :N], absref + resid.double()[:, :N].abs()
  fields = dict(a1=A.half() if f16 else A, c1=K, conv=0, taps=1, f16=int(f16), a_rows=a_rows, a_ld=lda, a_batch_rows=abr,
                wt=Wm.half() if f16 else Wm, n_total=N, k_total=K, w_rows=w_rows, w_ld=ldw, w_batch_rows=wbr, nbatch=nb,
                m_per_batch=M, bias=bias, rowvec=rowvec, rowvec_ld=N, residual=resid, ld_res=ldr if res else 0,
                rows_per_img=T)
  form = 'single256' if N == 256 and nb * ((M + 127) // 128) > _sms() // 2 else 'single128'
  what = 'gemm nb{nb} M{M} N{N} K{K} T{T}'.format(**case) + (' f16' if f16 else ' tf32') + (' +res' if res else '')
  _run_modes(dev, what, fields, ref, absref, K + 4, rows, N, N, img, nimg, form)


def _sms():
  import ctypes
  n = ctypes.c_int(0)
  _lib.call('b200_device_sm_count', ctypes.byref(n))
  return n.value


# ---------------------------------------------------------------------------------------------------------------------
# b. network heads
# ---------------------------------------------------------------------------------------------------------------------
SIGMAS = [0.37, 5.5, 0.011]


def _divisors(kind, B, dev):
  """(tensor, stride, per-image values) of a per-image, uniform or absent divisor.  The uniform table holds other
  values past its first entry, which a head that ignored div_stride would read."""
  if kind == 'none':
    return None, 0, torch.ones(B, device=dev, dtype=torch.float64)
  if kind == 'img':
    d = torch.tensor(SIGMAS[:B], device=dev)
    return d, 1, d.double()
  d = torch.tensor([SIGMAS[0], 1000.0, 3.0], device=dev)
  return d, 0, d.double()[:1].expand(B)


@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('R', [16, 32, 64, 256])
def test_tensor_core_nchw_head(dev, R, B, f16):
  C = 128
  g = _gen(dev, 31)
  x, x64 = _grid(torch.randn(B, R, R, C, device=dev, generator=g), f16)
  wt, w64 = _grid(torch.randn(128, C, 3, 3, device=dev, generator=g) / np.sqrt(9 * C), f16)
  import gpu_util
  wp = gpu_util.pack_conv_weight(wt.float(), f16=f16)        # all 128 rows nonzero: padded rows must not reach the output
  bias = torch.randn(128, device=dev, generator=g)
  conv = _conv64(x64, w64[:32]).permute(0, 3, 1, 2)              # [B][32][R][R]
  absconv = _conv64(x64.abs(), w64[:32].abs()).permute(0, 3, 1, 2)
  form = 'swap-halo' if R in (16, 32) else 'swap'
  for n_valid in (1, 3, 32):
    for kind in ('img', 'uniform', 'none'):
      div, stride, dv = _divisors(kind, B, dev)
      n = B * n_valid * R * R
      out = _out(n, 0, dev)
      got = _tc(dev, a1=x, c1=C, conv=1, h=R, w=R, nimg=B, taps=9, f16=int(f16), wt=wp, n_total=128, k_total=C,
                w_rows=9 * 128, nbatch=1, bias=bias, rows_per_img=R * R, out=out, ld_out=128, out_nchw=1,
                n_valid=n_valid, per_img_div=div, div_stride=stride)
      torch.cuda.synchronize()
      what = f'head {R}x{R} B{B} n_valid {n_valid} div {kind}' + (' f16' if f16 else ' tf32')
      assert got == form, f'{what}: form {got!r}'
      _check_sentinel(out, n, what)
      b64 = bias.double()[:n_valid].view(1, -1, 1, 1)
      d = dv.view(-1, 1, 1, 1)
      ref = (conv[:, :n_valid] + b64) / d
      absref = (absconv[:, :n_valid] + b64.abs()) / d.abs()
      _check_bound(what, out[:n].view(B, n_valid, R, R), ref, absref, 9 * C + 3, 0)


SMALL_N = [(N, C, f16) for N in (1, 3, 4) for C in (16, 128, 512) for f16 in (False, True) if not (f16 and C % 64)]


@pytest.mark.parametrize('N,C,f16', SMALL_N, ids=lambda v: str(v))
def test_cuda_core_small_n_head(dev, N, C, f16):
  B, H, W = 3, 15, 9                                             # odd sizes: partial warps, ragged borders
  g = _gen(dev, 32)
  x = torch.randn(B, H, W, C, device=dev, generator=g)
  if f16:
    x = x.half()
  x64 = x.double()
  wt = torch.randn(N, C, 3, 3, device=dev, generator=g) / np.sqrt(9 * C)
  import gpu_util
  wp = gpu_util.pack_conv_weight(wt)                            # [9][N][C] fp32, exact copy
  bias = torch.randn(N, device=dev, generator=g)
  conv = _conv64(x64, wt.double()).permute(0, 3, 1, 2)
  absconv = _conv64(x64.abs(), wt.double().abs()).permute(0, 3, 1, 2)
  for kind in ('img', 'uniform', 'none'):
    div, stride, dv = _divisors(kind, B, dev)
    n = B * N * H * W
    out = _out(n, 0, dev)
    _lib.call('b200_head_small_n_f32', _lib.ptr(x), int(f16), B, H, W, C, _lib.ptr(wp), _lib.ptr(bias), N, _lib.ptr(div),
              stride, _lib.ptr(out), _lib.stream_ptr(dev))
    torch.cuda.synchronize()
    what = f'small_n N{N} C{C} div {kind}' + (' f16' if f16 else ' fp32')
    _check_sentinel(out, n, what)
    d = dv.view(-1, 1, 1, 1)
    ref = (conv + bias.double().view(1, -1, 1, 1)) / d
    absref = (absconv + bias.double().abs().view(1, -1, 1, 1)) / d.abs()
    # fp32 FMAs: 9C products per output, folded over up to 8 lanes, + bias, / sigma
    _check_bound(what, out[:n].view(B, N, H, W), ref, absref, 9 * C + 8, 0)


# ---------------------------------------------------------------------------------------------------------------------
# c. stride-2 VALID convolutions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cout', [128, 256])
@pytest.mark.parametrize('f16', [False, True], ids=['tf32', 'f16'])
@pytest.mark.parametrize('B,H', [(1, 128), (2, 32), (4, 16), (8, 8), (9, 4)], ids=lambda v: str(v))
def test_stride2_valid_conv(dev, B, H, f16, cout):
  C, Hin = 128, 2 * H
  g = _gen(dev, 41)
  x, x64 = _grid(torch.randn(B, Hin, Hin, C, device=dev, generator=g), f16)
  wt, w64 = _grid(torch.randn(cout, C, 3, 3, device=dev, generator=g) / np.sqrt(9 * C), f16)
  import gpu_util
  wp = gpu_util.pack_conv_weight(wt.float(), f16=f16)
  bias = torch.randn(cout, device=dev, generator=g)
  M, HW = B * H * H, H * H
  ref = _conv64(x64, w64, 2, valid_pad=True).reshape(M, cout) + bias.double()
  absref = _conv64(x64.abs(), w64.abs(), 2, valid_pad=True).reshape(M, cout) + bias.double().abs()
  img = torch.arange(M, device=dev) // HW
  for stats in (False, True):
    mode = 1 if stats else (2 if f16 else 0)
    out = _out(M * cout, mode, dev)
    q = _qbuf(B, cout, dev) if stats else None
    got = _tc(dev, a1=x, c1=C, conv=1, h=H, w=H, nimg=B, taps=9, stride=2, valid_pad=1, hin=Hin, win=Hin, f16=int(f16),
              wt=wp, n_total=cout, k_total=C, w_rows=9 * cout, nbatch=1, bias=bias, rows_per_img=HW, out=out, ld_out=cout,
              store_mode=mode, qstats=q)
    torch.cuda.synchronize()
    what = f'stride2 B{B} {Hin}->{H} ->{cout}' + (' f16' if f16 else ' tf32') + (' +stats' if stats else '')
    assert got.startswith('single'), f'{what}: form {got!r}'
    _check_sentinel(out, M * cout, what)
    y = out[:M * cout].view(M, cout)
    _check_bound(what, y, ref, absref, 9 * C + 2, mode)
    if stats:
      _check_stats(what, q, y, img, B, cout)


# ---------------------------------------------------------------------------------------------------------------------
# d. split TF32
# ---------------------------------------------------------------------------------------------------------------------
def _split(t):
  import gpu_util
  hi = gpu_util.round_tf32(t)
  return hi, gpu_util.round_tf32(t - hi)


def _rel(y, ref):
  return ((y.double() - ref).norm() / ref.norm()).item()


SPLIT_CONV = [
    dict(B=2, H=32, W=32, C=128, N=128, k=3, skip=(), form='swap-halo'),
    dict(B=160, H=8, W=8, C=128, N=256, k=3, skip=(), form='single256'),
    dict(B=9, H=4, W=4, C=256, N=256, k=3, skip=(), form='single128'),
    dict(B=2, H=16, W=16, C=64, N=128, k=1, skip=(64, 32), form='swap'),     # extra 1x1 phase from two skip sources
]


def _split_compare(what, run, ref):
  """run(split) -> output: split TF32 within 1e-5 rel-L2 of float64, and at least 20x closer than plain TF32 on the same
  (RNA-rounded hi) operands."""
  e3, e1 = _rel(run(True), ref), _rel(run(False), ref)
  print(f'[split] {what}: rel-L2 3xtf32 {e3:.3e} (bound 1e-5: {e3 / 1e-5:.3e}), tf32 {e1:.3e}, ratio {e1 / max(e3, 1e-30):.1f}')
  assert e3 <= 1e-5, f'{what}: split TF32 rel-L2 {e3:.3g}'
  assert e3 * 20 <= e1, f'{what}: split TF32 ({e3:.3g}) not 20x better than TF32 ({e1:.3g})'


@pytest.mark.parametrize('case', SPLIT_CONV, ids=lambda c: 'B{B}_{H}x{W}_{C}-{N}_k{k}'.format(**c) + ('_skip' if c['skip'] else ''))
def test_split_tf32_conv(dev, case):
  B, H, W, C, N, k, skip = (case[x] for x in ('B', 'H', 'W', 'C', 'N', 'k', 'skip'))
  g = _gen(dev, 51)
  import gpu_util
  x = torch.randn(B, H, W, C, device=dev, generator=g)
  wt = torch.randn(N, C, k, k, device=dev, generator=g) / np.sqrt(k * k * C)
  wp = gpu_util.pack_conv_weight(wt)
  bias = torch.randn(N, device=dev, generator=g)
  M = B * H * W
  ref = _conv64(x.double(), wt.double()).reshape(M, N) + bias.double()
  xs, ws = _split(x), _split(wp)
  extra, extra_lo = {}, {}
  if skip:
    s = [torch.randn(B, H, W, c, device=dev, generator=g) for c in skip]
    w2 = torch.randn(N, sum(skip), device=dev, generator=g) / np.sqrt(sum(skip))
    ref = ref + torch.cat(s, 3).double().reshape(M, -1) @ w2.double().t()
    ss, w2s = [_split(t) for t in s], _split(w2)
    extra = dict(a3=ss[0][0], c3=skip[0], a4=ss[1][0], c4=skip[1], w2=w2s[0])
    extra_lo = dict(a3_lo=ss[0][1], a4_lo=ss[1][1], w2_lo=w2s[1])

  def run(split):
    out = _out(M * N, 0, dev)
    lo = dict(split=1, a1_lo=xs[1], w_lo=ws[1], **extra_lo) if split else {}
    got = _tc(dev, a1=xs[0], c1=C, conv=1, h=H, w=W, nimg=B, taps=k * k, wt=ws[0], n_total=N, k_total=C, w_rows=k * k * N,
              nbatch=1, bias=bias, rows_per_img=H * W, out=out, ld_out=N, **extra, **lo)
    torch.cuda.synchronize()
    assert got == case['form'] + (' 3xtf32' if split else ''), got
    _check_sentinel(out, M * N, 'split conv')
    return out[:M * N].view(M, N)
  _split_compare('B{B} {H}x{W} {C}->{N} k{k}'.format(**case) + (' +skip' if skip else ''), run, ref)


def test_split_tf32_batched_gemm(dev):
  nb, M, N, K, lda, ldw = 2, 256, 256, 128, 160, 192
  g = _gen(dev, 52)
  A = torch.randn(nb * M, lda, device=dev, generator=g)
  Wm = torch.randn(nb * N, ldw, device=dev, generator=g) / np.sqrt(K)
  bias = torch.randn(N, device=dev, generator=g)
  ref = torch.cat([A.double()[b * M:(b + 1) * M, :K] @ Wm.double()[b * N:(b + 1) * N, :K].t() for b in range(nb)]) + bias.double()
  As, Ws = _split(A), _split(Wm)

  def run(split):
    out = _out(nb * M * N, 0, dev)
    lo = dict(split=1, a1_lo=As[1], w_lo=Ws[1]) if split else {}
    _tc(dev, a1=As[0], c1=K, conv=0, taps=1, a_rows=nb * M, a_ld=lda, a_batch_rows=M, wt=Ws[0], n_total=N, k_total=K,
        w_rows=nb * N, w_ld=ldw, w_batch_rows=N, nbatch=nb, m_per_batch=M, bias=bias, rows_per_img=M, out=out, ld_out=N, **lo)
    torch.cuda.synchronize()
    _check_sentinel(out, nb * M * N, 'split gemm')
    return out[:nb * M * N].view(nb * M, N)
  _split_compare('gemm nb2 256x256x128 pitched', run, ref)


# ---------------------------------------------------------------------------------------------------------------------
# e. few-channel convolution: GroupNorm+SiLU on load, output quad sums
# ---------------------------------------------------------------------------------------------------------------------
def _gn_apply_takes_stream_path(C):
  """launch_gn_apply's choice for an fp32 input: the streaming kernel (whose arithmetic gn_coeff reproduces) when a CTA
  of 128..384 threads in steps of 32 holds a whole number of channel quads."""
  Q = C // 4
  threads = next((t for t in range(128, 385, 32) if t % Q == 0), 384)
  return threads % Q == 0 and Q <= 128


LOWC = [
    dict(B=20, H=64, W=64, C1=16, C2=0, N=16, k=3, G=4),        # 320 tiles on 2 CTAs per SM: CTAs cross images
    dict(B=2, H=32, W=32, C1=32, C2=16, N=32, k=3, G=12),       # two sources
    dict(B=2, H=32, W=64, C1=64, C2=0, N=64, k=3, G=16),        # weight slabs re-staged per work item
    dict(B=2, H=16, W=32, C1=128, C2=64, N=64, k=3, G=16),      # 12-channel groups straddle the two sources
    dict(B=2, H=32, W=32, C1=32, C2=16, N=16, k=1, G=12),
]


@pytest.mark.parametrize('mode', [0, 1], ids=['fp32', 'tf32'])
@pytest.mark.parametrize('case', LOWC, ids=lambda c: 'B{B}_{H}x{W}_{C1}+{C2}-{N}_k{k}_G{G}'.format(**c))
def test_conv_lowc_groupnorm_on_load(dev, case, mode):
  B, H, W, C1, C2, N, k, G = (case[x] for x in ('B', 'H', 'W', 'C1', 'C2', 'N', 'k', 'G'))
  C, HW, M = C1 + C2, H * W, B * H * W
  assert _gn_apply_takes_stream_path(C)
  g = _gen(dev, 61)
  x1 = torch.randn(B, H, W, C1, device=dev, generator=g) * 2 + 0.5
  x2 = torch.randn(B, H, W, C2, device=dev, generator=g) * 2 - 0.5 if C2 else None
  gamma = torch.randn(C, device=dev, generator=g) * 0.5 + 1
  beta = torch.randn(C, device=dev, generator=g) + 4            # a padding ring holding silu(shift) would add ~4 per tap
  import gpu_util
  wt = gpu_util.round_tf32(torch.randn(N, C, k, k, device=dev, generator=g) / np.sqrt(k * k * C))
  wp = gpu_util.pack_conv_weight(wt)
  bias = torch.randn(N, device=dev, generator=g)
  rowvec = torch.randn(B, N, device=dev, generator=g)
  resid = torch.randn(B, H, W, N, device=dev, generator=g)
  scale = 0.7071067690849304
  # the engine's two launches: GroupNorm statistics, then the normalised tensor in TF32-grid mode
  qws = torch.zeros(B * C // 4 * 2, device=dev, dtype=torch.float64)
  y = torch.empty(B, H, W, C, device=dev)
  _lib.call('b200_groupnorm_nhwc_f32', _lib.ptr(x1), C1, _lib.ptr(x2), C2, _lib.ptr(gamma), _lib.ptr(beta), B, HW, G,
            1e-6, 1, 1, _lib.ptr(qws), _lib.ptr(y), None, _lib.stream_ptr(dev))
  q1, q2 = qws[:B * C1 // 4 * 2], (qws[B * C1 // 4 * 2:] if C2 else None)
  plain = gpu_util.conv_nhwc(y, None, wp, bias, N, k, rowvec=rowvec, rowvec_ld=N, residual=resid, scale=scale,
                             round_out=mode, impl=3)
  coeff = torch.full((2 * B * C + 64,), SENT, device=dev)
  out = _out(M * N, mode, dev)
  q = _qbuf(B, N, dev)
  _lib.call('b200_conv_lowc_gn_f32', _lib.ptr(x1), C1, _lib.ptr(x2), C2, B, H, W, _lib.ptr(wp), N, k, _lib.ptr(q1),
            _lib.ptr(q2), _lib.ptr(gamma), _lib.ptr(beta), G, 1e-6, 1, _lib.ptr(coeff), _lib.ptr(bias), _lib.ptr(rowvec), N,
            _lib.ptr(resid), scale, mode, _lib.ptr(out), _lib.ptr(q), _lib.stream_ptr(dev))
  torch.cuda.synchronize()
  what = 'lowc B{B} {H}x{W} {C1}+{C2}->{N} k{k} G{G}'.format(**case) + f' mode {mode}'
  _check_sentinel(out, M * N, what)
  got = out[:M * N].view(B, H, W, N)
  assert torch.equal(got, plain), f'{what}: GroupNorm on load differs from the normalised tensor by ' \
                                  f'{(got - plain).abs().max().item():.3g}'
  y64 = y.double()
  img = torch.arange(M, device=dev) // HW
  ref = ((_conv64(y64, wt.double()) + bias.double() + rowvec.double()[:, None, None, :] + resid.double()) * scale)
  absref = ((_conv64(y64.abs(), wt.double().abs()) + bias.double().abs() + rowvec.double().abs()[:, None, None, :] +
             resid.double().abs()) * scale)
  _check_bound(what, got.reshape(M, N), ref.reshape(M, N), absref.reshape(M, N), k * k * C + 4, mode)
  _check_stats(what, q, got.reshape(M, N), img, B, N)
