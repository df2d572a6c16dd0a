"""`-m gpu`: the NCSNv2 family (configs/ve/ncsnv2/*.py) on the engine.  Its kernels against float64 references
(InstanceNorm2dPlus + ELU in every store format, the dilated convolution on the tensor cores and the CUDA cores, the CRP
max pool, the MSF bilinear sum), whole networks against the oracle, and the discrete-time ALD sampler on the host loop
against the reference's own draws (tests/golden/pc_ncsnv2_tiny.npz)."""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import pack_conv_weight, round_tf32, strict_fp32, to_nchw, to_nhwc
from helpers import golden, rel_l2
from ncsnv2_helpers import golden_config, seeded_ncsnv2
from oracle import ncsnv2_oracle as VO
from score_sde_pytorch_b200 import _lib

pytestmark = pytest.mark.gpu

MODES = {0: torch.float32, 1: torch.float32, 2: torch.float16}   # store formats: fp32, TF32 grid, fp16


@pytest.fixture(scope='module')
def dev():
  strict_fp32()
  return torch.device('cuda:0')


def _sd64(model, dev):
  return {k: v.to(dev).double() for k, v in model.state_dict().items()}


def _in_plus64(x, alpha, gamma, beta):
  p = {'n.alpha': alpha.double(), 'n.gamma': gamma.double(), 'n.beta': beta.double()}
  return VO.in_plus(x.double(), p, 'n')


# ---- kernels ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('case', ['random', 'equal_means'])
@pytest.mark.parametrize('B,C,H', [(3, 128, 16), (2, 256, 64), (1, 128, 128)])
def test_instance_norm_plus_elu_matches_float64(dev, mode, case, B, C, H):
  """16x16 images are summed by one pixel slice per CTA column, 64x64 and 128x128 ones by 8 and 32 slices."""
  torch.manual_seed(11)
  W = H
  x = torch.randn(B, C, H, W, device=dev) * 2
  if case == 'random':
    x += torch.randn(1, C, 1, 1, device=dev) * 3
  else:   # channel means equal to 1e-6: v is tiny, and eps decides (mu - m) / sqrt(v + eps)
    x = x - x.mean(dim=(2, 3), keepdim=True) + 0.75 + 1e-6 * torch.randn(B, C, 1, 1, device=dev)
  alpha, gamma = 1 + 0.3 * torch.randn(C, device=dev), 1 + 0.3 * torch.randn(C, device=dev)
  beta = 0.2 * torch.randn(C, device=dev)
  stats = torch.empty(B * C * 66, dtype=torch.float64, device=dev)
  xin = to_nhwc(x)   # (every operand is held by a name until the kernel has read it)
  for act in (0, 1):
    y = torch.empty(B, H, W, C, dtype=MODES[mode], device=dev)
    _lib.call('b200_instnorm_plus_nhwc_f32', _lib.ptr(xin), B, H * W, C, _lib.ptr(alpha), _lib.ptr(gamma),
              _lib.ptr(beta), act, mode, _lib.ptr(y), _lib.ptr(stats), _lib.stream_ptr(dev))
    ref = _in_plus64(x, alpha, gamma, beta)
    if act:
      ref = F.elu(ref)
    e = rel_l2(to_nchw(y.float()), ref)
    print(f'in++ {case} {B}x{C}x{H}x{W} act={act} mode={mode}: rel-L2 {e:.2e}')
    assert e < (2e-6 if mode == 0 else 1e-3)


@pytest.mark.parametrize('dil', [2, 4])
@pytest.mark.parametrize('B', [1, 3, 37])
@pytest.mark.parametrize('impl', [0, 1, 2])
@pytest.mark.parametrize('C,N', [(128, 128), (256, 256)])
def test_dilated_conv_matches_float64_with_borders(dev, dil, B, impl, C, N):
  """3x3 'same' convolution with taps `dil` pixels apart on 16x16 images; the border rows / columns (where taps read the
  zero padding) are checked on their own as well as the whole output.  128 output channels take the swapped tensor-core
  form, 256 (the network's dilated blocks) the row-major one."""
  torch.manual_seed(12 + dil + B)
  H = 16
  x = torch.randn(B, C, H, H, device=dev)
  w = torch.randn(N, C, 3, 3, device=dev) / (3 * C ** 0.5)
  b = torch.randn(N, device=dev)
  res = torch.randn(B, N, H, H, device=dev)
  xin = to_nhwc(x)
  if impl == 1:
    xin = round_tf32(xin)
  if impl == 2:
    xin = xin.half()
  wp = pack_conv_weight(w, round_tf32_=impl == 1, f16=impl == 2)
  out = torch.empty(B, H, H, N, device=dev)
  res_nhwc = to_nhwc(res)
  _lib.call('b200_conv_dilated_nhwc_f32', _lib.ptr(xin), C, B, H, H, _lib.ptr(wp), _lib.ptr(b), N, dil,
            _lib.ptr(res_nhwc), 0, _lib.ptr(out), impl, _lib.stream_ptr(dev))
  ref = F.conv2d(x.double(), w.double(), b.double(), padding=dil, dilation=dil) + res.double()
  got = to_nchw(out)
  tol = 1e-6 if impl == 0 else 2e-3
  e = rel_l2(got, ref)
  border = torch.zeros(H, H, dtype=torch.bool, device=dev)
  border[:dil], border[-dil:], border[:, :dil], border[:, -dil:] = True, True, True, True
  eb = rel_l2(got[:, :, border].unsqueeze(-1), ref[:, :, border].unsqueeze(-1))
  print(f'dilated conv {C}->{N} d={dil} B={B} impl={impl}: rel-L2 {e:.2e}, border {eb:.2e}')
  assert e < tol and eb < tol


@pytest.mark.parametrize('mode', [0, 1, 2])
def test_maxpool5_matches_torch_with_borders_and_sum(dev, mode):
  torch.manual_seed(13)
  B, C, H, W = 2, 64, 16, 8
  x = torch.randn(B, C, H, W, device=dev) - 3.0   # all negative near the borders: a zero padding would show
  add = torch.randn(B, C, H, W, device=dev)
  y = torch.empty(B, H, W, C, dtype=MODES[mode], device=dev)
  s = torch.empty(B, H, W, C, device=dev)
  x_nhwc, add_nhwc = to_nhwc(x), to_nhwc(add)
  _lib.call('b200_maxpool5_nhwc_f32', _lib.ptr(x_nhwc), B, H, W, C, mode, _lib.ptr(y), _lib.ptr(add_nhwc),
            _lib.ptr(s), _lib.stream_ptr(dev))
  ref = F.max_pool2d(x.double(), kernel_size=5, stride=1, padding=2)
  got = to_nchw(y.float()).double()
  if mode == 0:
    assert torch.equal(got, ref)
  else:
    assert rel_l2(got, ref) < 1e-3
  assert torch.equal(to_nchw(s), x + add)


@pytest.mark.parametrize('shape', [(16, 32), (8, 16), (32, 64)])
def test_bilinear_add_matches_float64(dev, shape):
  torch.manual_seed(14)
  lo_h, hi_h = shape
  B, C = 3, 64
  lo = torch.randn(B, C, lo_h, lo_h, device=dev)
  acc = torch.randn(B, C, hi_h, hi_h, device=dev)
  out, lo_nhwc = to_nhwc(acc), to_nhwc(lo)
  _lib.call('b200_bilinear_add_nhwc_f32', _lib.ptr(lo_nhwc), B, lo_h, lo_h, C, _lib.ptr(out), hi_h, hi_h,
            _lib.stream_ptr(dev))
  ref = acc.double() + F.interpolate(lo.double(), size=(hi_h, hi_h), mode='bilinear', align_corners=True)
  e = rel_l2(to_nchw(out), ref)
  print(f'bilinear add {lo_h}->{hi_h}: rel-L2 {e:.2e}')
  assert e < 1e-6


# ---- whole networks -----------------------------------------------------------------------------------------------------
def test_tiny_network_every_block_fp32(dev):
  g = golden('ncsnv2_tiny.npz')
  cfg = golden_config('tiny')
  model = seeded_ncsnv2(cfg, precision='fp32', keep_activations=True).to(dev)
  x, y = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['y']).to(dev)
  out = model(x, y)
  taps = {}
  with torch.no_grad():
    ref = VO.ncsnv2_forward(_sd64(model, dev), cfg, x.double(), y, taps=taps)
  assert out.dtype == torch.float64
  for i, name in enumerate(model.tap_names()):
    e = rel_l2(model.tap(i), taps[i])
    print(f'tiny fp32 block {i} {name}: rel-L2 {e:.2e}')
    assert e < 1e-5, name
  e = rel_l2(out, ref)
  print(f'tiny fp32 output: rel-L2 {e:.2e} (vs the reference fixture {rel_l2(out.cpu(), torch.from_numpy(g["out"])):.2e})')
  assert e < 1e-5 and rel_l2(out.cpu(), torch.from_numpy(g['out'])) < 1e-5


@pytest.mark.parametrize('name,batch', [('cifar10', 4), ('celeba', 1), ('bedroom', 1)])
@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'f16'])
def test_full_size_network_matches_oracle(dev, name, batch, precision):
  cfg = golden_config(name)
  model = seeded_ncsnv2(cfg, precision=precision).to(dev)
  torch.manual_seed(21)
  R = cfg.data.image_size
  x = torch.rand(batch, 3, R, R, device=dev)
  y = torch.tensor([5, 40, cfg.model.num_scales // 2, cfg.model.num_scales - 1][:batch], device=dev)
  out = model(x, y)
  with torch.no_grad():
    ref = VO.ncsnv2_forward(_sd64(model, dev), cfg, x.double(), y)
  e = rel_l2(out, ref)
  print(f'{name} batch {batch} [{precision}]: per-image rel-L2 vs oracle {e:.3e}')
  assert out.dtype == torch.float64 and out.shape == x.shape
  assert e < (1e-5 if precision == 'fp32' else 2.5e-3)


def test_forward_is_deterministic_and_tf32_plan_runs_on_tensor_cores(dev):
  cfg = golden_config('cifar10')
  model = seeded_ncsnv2(cfg, precision='tf32').to(dev)
  torch.manual_seed(22)
  x = torch.rand(8, 3, 32, 32, device=dev)
  y = torch.arange(8, device=dev) * 20
  a, b = model(x, y), model(x, y)
  assert torch.equal(a, b)
  names = model.op_names()
  assert any('d2' in n and 'swap' in n or 'd2' in n and 'single' in n for n in names)   # dilated 3x3 on the tensor cores
  assert any('d4' in n for n in names) and any('maxpool5x5' in n for n in names) and any('bilinear' in n for n in names)
  assert not any('cuda-core' in n and n.startswith('conv3x3 128') for n in names)


@pytest.mark.parametrize('name,batch,keep', [('tiny', 2, True), ('cifar10', 4, True), ('cifar10', 4, False), ('bedroom', 1, True)])
def test_forward_writes_nothing_past_its_workspace(dev, name, batch, keep):
  """The plan is bound to a workspace of exactly b200_ncsnpp_workspace_bytes, followed by guard words; a forward leaves the
  guard as it was.  keep_activations=True stacks every buffer, so the last one planned ends at the top of the workspace."""
  cfg = golden_config(name)
  model = seeded_ncsnv2(cfg, precision='tf32', keep_activations=keep).to(dev)
  eng = model.engine(batch, dev)
  lib = _lib.load()
  need = lib.b200_ncsnpp_workspace_bytes(eng['h'], batch)
  guard = 1 << 16
  ws = torch.full((need // 4 + guard,), 12345.0, device=dev)
  _lib.call('b200_ncsnpp_bind_workspace', eng['h'], batch, _lib.ptr(ws), need)
  eng['ws'] = ws
  torch.manual_seed(23)
  R = cfg.data.image_size
  x = torch.rand(batch, 3, R, R, device=dev)
  out = model(x, torch.arange(batch, device=dev))
  torch.cuda.synchronize()
  assert torch.isfinite(out).all()
  assert bool((ws[-guard:] == 12345.0).all()), 'the forward wrote past the end of its workspace'


# ---- sampling -----------------------------------------------------------------------------------------------------------
class _OnDevice(torch.nn.Module):
  """The engine network behind a host-side sampler: inputs to the GPU, the float64 output back to the host."""

  def __init__(self, net, dev):
    super().__init__()
    self.net, self.dev = net, dev

  def forward(self, x, y):
    return self.net(x.to(self.dev), y.to(self.dev)).cpu()


def test_tiny_ald_host_loop_matches_reference_draw_for_draw(dev):
  """configs/ve/ncsnv2: predictor 'none', corrector 'ald', continuous=False.  The sampler's noise is drawn on the host
  with the reference's seed, so each Langevin step sees the reference's draw; the network runs on the engine (fp32)."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  g = golden('pc_ncsnv2_tiny.npz')
  cfg = golden_config('tiny')
  model = seeded_ncsnv2(cfg, precision='fp32').to(dev)
  sde = sde_lib.VESDE(sigma_min=cfg.model.sigma_min, sigma_max=cfg.model.sigma_max, N=20)
  shape = g['ald'].shape
  assert native.match_pc_plan(sde=sde, model=model, predictor=sampling.NonePredictor,
                              corrector=sampling.AnnealedLangevinDynamics, shape=shape, snr=cfg.sampling.snr, n_steps=2,
                              probability_flow=False, continuous=False, eps=1e-5, device=dev) is None   # the host loop
  fn = sampling.get_pc_sampler(sde, shape, sampling.NonePredictor, sampling.AnnealedLangevinDynamics, lambda v: v,
                               snr=cfg.sampling.snr, n_steps=2, probability_flow=False, continuous=False, denoise=True,
                               eps=1e-5, device='cpu')
  torch.manual_seed(44)
  s, nfe = fn(_OnDevice(model, dev))
  e = rel_l2(s, torch.from_numpy(g['ald']))
  print(f'tiny ALD host loop (N=20, 2 steps per level, fp32): rel-L2 vs reference {e:.3e}, nfe {nfe}')
  assert nfe == int(g['ald_nfe'])
  assert str(s.dtype) == str(g['ald_dtype'])
  assert e < 1e-4


def test_ald_sampler_on_device_is_deterministic(dev):
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_ncsnv2(cfg, precision='tf32').to(dev)
  sde = sde_lib.VESDE(sigma_min=cfg.model.sigma_min, sigma_max=cfg.model.sigma_max, N=20)
  fn = sampling.get_pc_sampler(sde, (4, 3, 16, 16), sampling.NonePredictor, sampling.AnnealedLangevinDynamics, lambda v: v,
                               snr=cfg.sampling.snr, n_steps=2, probability_flow=False, continuous=False, denoise=True,
                               eps=1e-5, device=dev)
  runs = []
  for _ in range(2):
    torch.manual_seed(45)
    runs.append(fn(model)[0])
  assert runs[0].dtype == torch.float64 and torch.isfinite(runs[0]).all()
  assert torch.equal(runs[0], runs[1])


def test_continuous_time_paths_refuse(dev):
  """The native PC loop, the ODE sampler and the likelihood feed time / sigma labels; NCSNv2 takes indices."""
  from score_sde_pytorch_b200 import likelihood, sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_ncsnv2(cfg).to(dev)
  sde = sde_lib.VESDE(N=20)
  fn = sampling.get_pc_sampler(sde, (1, 3, 16, 16), sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector,
                               lambda v: v, snr=0.16, continuous=True, device=dev)
  with pytest.raises(TypeError, match='noise-level indices'):
    fn(model)
  with pytest.raises(NotImplementedError, match='noise-level indices'):
    sampling.get_ode_sampler(sde, (1, 3, 16, 16), lambda v: v, device=dev)(model)
  with pytest.raises(NotImplementedError, match='NCSNv2'):
    likelihood.get_likelihood_fn(sde, lambda v: v)(model, torch.rand(1, 3, 16, 16, device=dev))
