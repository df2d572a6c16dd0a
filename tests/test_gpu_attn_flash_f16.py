"""`-m gpu`: the flash fp16 attention core (attn_flash.cu) alone against a float64 torch reference on the same fp16
operands, then `precision='f16'` networks whose attention runs on it against the strict-fp32 oracle: one evaluation of
each test network and the native PC loop."""
import pytest
import torch

from ddpm_helpers import seeded_ddpm
from helpers import seeded_model, rel_l2
from oracle import ddpm_oracle as DO
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO
from score_sde_pytorch_b200 import _lib, configs

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3            # bound on SAMPLER outputs
TOL_SINGLE_EVAL_TC = 2.5e-3  # one network evaluation in a tensor-core mode (11-bit operand rounding through the chain)
TOL_CORE = 3e-4              # the core alone: P and the stored O are rounded to fp16


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _flash(qk, vT, bv):
  """qk [nimg*T, 2C] fp16, vT [nimg, C, T] fp16, bv [C] fp32 -> O [nimg*T, C] fp16."""
  nimg, C, T = vT.shape
  out = torch.empty(nimg * T, C, device=qk.device, dtype=torch.float16)
  _lib.call('b200_attention_flash_f16', _lib.ptr(qk), _lib.ptr(vT), _lib.ptr(bv), _lib.ptr(out), nimg, T, C,
            _lib.stream_ptr(qk.device))
  return out


def _reference(qk, vT, bv):
  """softmax(q k^T / sqrt(C)) v + b_v in float64, one image at a time (T = 4096: 128 MB of logits per image)."""
  nimg, C, T = vT.shape
  q = qk[:, :C].double().reshape(nimg, T, C)
  k = qk[:, C:].double().reshape(nimg, T, C)
  out = torch.empty(nimg, T, C, device=qk.device, dtype=torch.float64)
  for i in range(nimg):
    P = torch.softmax((q[i] @ k[i].t()) * (C ** -0.5), dim=-1)
    out[i] = P @ vT[i].double().t() + bv.double()
  return out.reshape(nimg * T, C)


def _inputs(nimg, T, C, seed, qscale=1.0):
  g = torch.Generator(device='cuda').manual_seed(seed)
  q = torch.randn(nimg, T, C, device='cuda', generator=g) * 1.5 * qscale
  k = torch.randn(nimg, T, C, device='cuda', generator=g) * 1.5
  v = torch.randn(nimg, T, C, device='cuda', generator=g)
  bv = torch.randn(C, device='cuda', generator=g)
  qk = torch.cat([q, k], 2).reshape(nimg * T, 2 * C).half().contiguous()
  vT = v.transpose(1, 2).half().contiguous()
  return qk, vT, bv


def _rel(a, b):
  return ((a.double() - b).norm() / b.norm()).item()


SHAPES = [(256, 128), (1024, 128), (1024, 256), (1024, 512), (4096, 128)]


@pytest.mark.parametrize('nimg', [1, 3, 37])
@pytest.mark.parametrize('T,C', SHAPES)
def test_flash_core_matches_float64(dev, T, C, nimg):
  """C <= 256: 128-row tiles, one warpgroup per 64 rows; C = 512: 64-row tiles, one warpgroup per 256 output channels.
  nimg = 37 puts several tiles on every CTA of the persistent grid (ring and Q-buffer reuse across tiles)."""
  qk, vT, bv = _inputs(nimg, T, C, seed=1000 * C + T + nimg)
  out = _flash(qk, vT, bv)
  torch.cuda.synchronize()
  assert torch.isfinite(out).all()
  err = _rel(out, _reference(qk, vT, bv))
  print(f'flash core T={T} C={C} nimg={nimg}: rel-L2 {err:.3e}')
  assert err < TOL_CORE, err
  # deterministic: no atomics, fixed order of every sum
  assert torch.equal(_flash(qk, vT, bv), out)


@pytest.mark.parametrize('T,C', SHAPES)
def test_flash_core_peaked_logits(dev, T, C):
  """q scaled 30x: the row max moves by hundreds between key blocks, so the running-max rescale of O and l decides the
  result (an unscaled exp() would overflow)."""
  qk, vT, bv = _inputs(3, T, C, seed=7 * T + C, qscale=30.0)
  out = _flash(qk, vT, bv)
  torch.cuda.synchronize()
  assert torch.isfinite(out).all()
  err = _rel(out, _reference(qk, vT, bv))
  print(f'flash core T={T} C={C}, peaked logits: rel-L2 {err:.3e}')
  assert err < TOL_CORE, err


NETWORKS = {
    'A_ddpmpp_T256_C128': ('ncsnpp', lambda: configs.tiny_ddpmpp(nf=64, image_size=32, ch_mult=(1, 2, 2), attn_resolutions=(16,)),
                           ['T=256 C=128']),
    'B_ncsnpp_T1024_C128': ('ncsnpp', lambda: configs.tiny_ncsnpp(nf=64, image_size=32, ch_mult=(2, 4), attn_resolutions=(32,)),
                            ['T=1024 C=128']),
    'C_ddpm_T1024_C128': ('ddpm', lambda: configs.tiny_ddpm(nf=64, image_size=64, ch_mult=(1, 2, 2, 2), attn_resolutions=(32,)),
                          ['T=1024 C=128']),
    'D_ddpm_T4096_C128': ('ddpm', lambda: configs.tiny_ddpm(nf=128, image_size=64, ch_mult=(1, 2), attn_resolutions=(64,)),
                          ['T=4096 C=128', 'T=1024 C=256']),
}


def _assert_flash(model, shapes):
  names = model.op_names()
  for s in shapes:
    assert any(f'attention flash {s}' in n and '[fused f16]' in n for n in names), names
  assert not any('softmax T=' in n for n in names), names


@pytest.mark.parametrize('name', sorted(NETWORKS))
def test_network_with_flash_attention_f16_matches_oracle(dev, name):
  family, cfg_fn, shapes = NETWORKS[name]
  cfg = cfg_fn()
  n = cfg.data.image_size
  model = (seeded_ddpm(cfg, precision='f16') if family == 'ddpm' else seeded_model(cfg, precision='f16')).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(8)
  if family == 'ddpm' or cfg.training.sde == 'vpsde':
    x = torch.randn(3, 3, n, n, device=dev)
    t = torch.tensor([17.0, 512.5, 940.0], device=dev)
  else:
    x = torch.randn(3, 3, n, n, device=dev) * 5
    t = torch.tensor([12.0, 0.9, 0.05], device=dev)
  with torch.no_grad():
    y = model(x, t)
    ref = DO.ddpm_forward(sd, cfg, x, t) if family == 'ddpm' else NO.ncsnpp_forward(sd, cfg, x, t)
  e = rel_l2(y, ref)
  print(f'{name} [f16]: rel-L2 vs oracle {e:.3e}')
  assert torch.isfinite(y).all()
  assert e < TOL_SINGLE_EVAL_TC
  _assert_flash(model, shapes)
  model._release()


def test_native_pc_loop_f16_with_flash_attention_matches_oracle(dev):
  """VE reverse diffusion + Langevin, 10 iterations on network B (attention at 32x32): the captured PC plan in f16."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  cfg = NETWORKS['B_ncsnpp_T1024_C128'][1]()
  shape = (3, 3, 32, 32)
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  torch.manual_seed(9)
  x0 = osde.prior_sampling(shape).to(dev)
  model = seeded_model(cfg, precision='f16').to(dev)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor, corrector=sampling.LangevinCorrector,
                              shape=shape, snr=0.16, n_steps=1, probability_flow=False, continuous=True, eps=1e-5, device=dev)
  assert plan is not None
  torch.cuda.manual_seed(78)
  _, xm = plan.run(x0, first_step=0, num_steps=10)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.cuda.manual_seed(78)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, eps=1e-5, device=dev, x_init=x0, num_iters=10)
  e = rel_l2(xm, ref)
  print(f'native PC loop, network B [f16]: rel-L2 vs oracle {e:.3e}')
  assert torch.isfinite(xm).all()
  assert e < TOL_PARITY
  _assert_flash(model, NETWORKS['B_ncsnpp_T1024_C128'][2])
