"""`-m gpu`: the fused fp16 attention core at T = 256 tokens x C = 512 channels (the 16x16 attention of the 256-pixel DDPM
configs and of FFHQ-1024 NCSN++), alone against torch on the same fp16 operands, then `precision='f16'` networks with
512-channel attention against the strict-fp32 oracle: tiny ones, the native PC loop, and the two reference configs."""
import pytest
import torch

from ddpm_helpers import golden_config as ddpm_config, seeded_ddpm
from helpers import golden_config, seeded_model, rel_l2
from oracle import ddpm_oracle as DO
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO
from score_sde_pytorch_b200 import configs

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3            # bound on SAMPLER outputs
TOL_SINGLE_EVAL_TC = 2.5e-3  # one network evaluation in a tensor-core mode (11-bit operand rounding through the chain)


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _torch_core(qk, vT, w3, bv, b3, x, sc):
  nimg, C, T = vT.shape
  q = qk[:, :C].float().reshape(nimg, T, C)
  k = qk[:, C:].float().reshape(nimg, T, C)
  P = torch.softmax(torch.bmm(q, k.transpose(1, 2)) * (C ** -0.5), dim=-1)
  h = torch.bmm(P, vT.float().transpose(1, 2)) + bv
  return ((h.reshape(nimg * T, C) @ w3.float().t() + b3) + x) * sc


@pytest.mark.parametrize('nimg', [1, 3, 150])
def test_fused_attention_core_f16_c512_matches_torch(dev, nimg):
  """C = 512: S = Q K^T over eight K blocks, E V and O' W3^T as two n256 halves each, 32 ring loads per tile.  nimg=150 ->
  300 tiles on the persistent grid (ring reuse across tiles)."""
  import gpu_util
  torch.manual_seed(41 + nimg)
  T, C = 256, 512
  q = (torch.randn(nimg, T, C, device=dev) * 1.5).half()
  k = (torch.randn(nimg, T, C, device=dev) * 1.5).half()
  v = torch.randn(nimg, T, C, device=dev).half()
  w3 = (torch.randn(C, C, device=dev) / 22).half()        # [out][in]
  bv, b3 = torch.randn(C, device=dev), torch.randn(C, device=dev)
  x = torch.randn(nimg * T, C, device=dev)
  qk = torch.cat([q, k], 2).reshape(nimg * T, 2 * C).contiguous()
  vT = v.transpose(1, 2).contiguous()
  sc = 0.7071067690849304
  out, qs = gpu_util.attention_core(qk, vT, w3, bv, b3, x, sc, want_stats=True)
  torch.cuda.synchronize()
  ref = _torch_core(qk, vT, w3, bv, b3, x, sc)
  err = ((out - ref).norm() / ref.norm()).item()
  assert err < 3e-4, err                                  # E and O' rounded to fp16 inside the chain
  # quad sums of what was stored, both 256-column halves of the output projection
  o4 = out.reshape(nimg, T, C // 4, 4).double()
  assert qs.shape == (nimg, C // 4, 2)
  assert torch.allclose(qs[..., 0], o4.sum((1, 3)), rtol=1e-5, atol=1e-3)
  assert torch.allclose(qs[..., 1], (o4 * o4).sum((1, 3)), rtol=1e-5, atol=1e-3)
  # peaked softmax rows (large logits): the max subtraction must keep exp() in range
  qk2 = (qk.float() * 6).half()
  out2 = gpu_util.attention_core(qk2, vT, w3, bv, b3, x, sc)
  ref2 = _torch_core(qk2, vT, w3, bv, b3, x, sc)
  assert torch.isfinite(out2).all()
  assert ((out2 - ref2).norm() / ref2.norm()).item() < 3e-4


def _tiny(family):
  """512 channels at 16x16 (nf = 128, ch_mult (1, 4)), 32x32 images."""
  if family == 'ddpm':
    return configs.tiny_ddpm(nf=128, image_size=32, ch_mult=(1, 4), attn_resolutions=(16,))
  return configs.tiny_ncsnpp(nf=128, image_size=32, ch_mult=(1, 4), attn_resolutions=(16,))


def _assert_fused_c512(model):
  names = model.op_names()
  assert any('attention core T=256 C=512' in n and '[fused]' in n for n in names), names
  assert not any('softmax T=256' in n for n in names), names


@pytest.mark.parametrize('family', ['ddpm', 'ncsnpp'])
def test_tiny_network_with_512_channel_attention_f16_matches_oracle(dev, family):
  cfg = _tiny(family)
  model = (seeded_ddpm(cfg, precision='f16') if family == 'ddpm' else seeded_model(cfg, precision='f16')).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(8)
  x = torch.randn(3, 3, 32, 32, device=dev) * (1 if family == 'ddpm' else 5)
  t = torch.tensor([17.0, 512.5, 940.0], device=dev) if family == 'ddpm' else torch.tensor([12.0, 0.9, 0.05], device=dev)
  with torch.no_grad():
    y = model(x, t)
    ref = DO.ddpm_forward(sd, cfg, x, t) if family == 'ddpm' else NO.ncsnpp_forward(sd, cfg, x, t)
  e = rel_l2(y, ref)
  print(f'tiny {family} C=512 attention [f16]: rel-L2 vs oracle {e:.3e}')
  assert torch.isfinite(y).all()
  assert e < TOL_SINGLE_EVAL_TC
  _assert_fused_c512(model)


def test_native_pc_loop_f16_with_512_channel_attention_matches_oracle(dev):
  """VE reverse diffusion + Langevin on the tiny NCSN++ with 512-channel attention: the captured PC plan in f16."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  cfg = _tiny('ncsnpp')
  shape = (3, 3, 32, 32)
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  torch.manual_seed(9)
  x0 = osde.prior_sampling(shape).to(dev)
  model = seeded_model(cfg, precision='f16').to(dev)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor, corrector=sampling.LangevinCorrector,
                              shape=shape, snr=0.16, n_steps=1, probability_flow=False, continuous=True, eps=1e-5, device=dev)
  assert plan is not None
  torch.cuda.manual_seed(78)
  _, xm = plan.run(x0, first_step=0, num_steps=4)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.cuda.manual_seed(78)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, eps=1e-5, device=dev, x_init=x0, num_iters=4)
  e = rel_l2(xm, ref)
  print(f'native PC loop, tiny NCSN++ C=512 attention [f16]: rel-L2 vs oracle {e:.3e}')
  assert torch.isfinite(xm).all()
  assert e < TOL_PARITY
  _assert_fused_c512(model)


def test_ddpm_celebahq_256_f16_matches_oracle(dev):
  """configs/vp/ddpm/celebahq.py (111.6 M parameters, 256x256), one evaluation at batch 1 in f16: the 16x16 512-channel
  attention on the fused core, the 8x8 one on the small-token core."""
  cfg = ddpm_config('celebahq_256')
  model = seeded_ddpm(cfg, precision='f16').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(3)
  x = torch.randn(1, 3, 256, 256, device=dev)
  labels = torch.tensor([417.3], device=dev)
  with torch.no_grad():
    y = model(x, labels)
    ref = DO.ddpm_forward(sd, cfg, x, labels)
  e = rel_l2(y, ref)
  print(f'ddpm celebahq-256 [f16] rel-L2 vs oracle {e:.3e}')
  assert torch.isfinite(y).all()
  assert e < TOL_SINGLE_EVAL_TC
  _assert_fused_c512(model)
  model._release()


def test_ffhq_1024_f16_matches_oracle(dev):
  """configs/ve/ffhq_ncsnpp_continuous.py (105.8 M parameters, 1024x1024), one evaluation at batch 1 in f16."""
  cfg = golden_config('ffhq_1024')
  model = seeded_model(cfg, precision='f16').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(4)
  x = torch.randn(1, 3, 1024, 1024, device=dev) * 5
  sigma = torch.tensor([3.0], device=dev)
  with torch.no_grad():
    y = model(x, sigma)
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma)
  e = rel_l2(y, ref)
  print(f'ffhq-1024 [f16] rel-L2 vs oracle {e:.3e}')
  assert torch.isfinite(y).all()
  assert e < TOL_SINGLE_EVAL_TC
  _assert_fused_c512(model)
  model._release()
