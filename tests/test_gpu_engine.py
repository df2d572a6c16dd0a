"""`-m gpu`: the NCSN++ engine (strict-fp32 execution mode) and the native PC loop against the oracle
on the same device, same weights, same seeds.  TF32 / fp16 tensor-core execution is covered in test_gpu_tc.py."""
import numpy as np
import pytest
import torch

from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _oracle_model(cfg, sd):
  return lambda x, labels: NO.ncsnpp_forward(sd, cfg, x, labels)


def _per_module_report(model, oracle_taps, limit=1e-4):
  rows = []
  for i in sorted(oracle_taps):
    try:
      mine = model.tap(i)
    except RuntimeError:
      continue
    rows.append((i, rel_l2(mine, oracle_taps[i])))
  bad = [r for r in rows if not (r[1] < limit)]
  return rows, bad


@pytest.mark.parametrize('name', ['tiny', 'tiny_noattn', 'tiny_vp'])
def test_forward_fp32_matches_oracle_and_reference_golden(dev, name):
  g = golden(f'ncsnpp_{name}.npz')
  cfg = golden_config(name)
  model = seeded_model(cfg, precision='fp32', keep_activations=True).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  x, sigma = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma, taps=taps)
    y = model(x, sigma)
  rows, bad = _per_module_report(model, taps)
  assert not bad, f'first diverging modules (index, rel-L2): {bad[:6]} of {len(rows)}'
  assert rel_l2(y, ref) < 1e-4
  assert rel_l2(y, torch.from_numpy(g['y']).to(dev)) < 1e-4    # the reference's own CPU output


def test_forward_batch_replan_and_uniform_labels(dev):
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(3)
  for B in (1, 5, 2):
    x = torch.randn(B, 3, 16, 16, device=dev) * 2
    sigma = torch.full((B,), 1.7, device=dev)
    with torch.no_grad():
      ref = NO.ncsnpp_forward(sd, cfg, x, sigma)
      y = model(x, sigma)
      yu = model(x, sigma, labels_uniform=True)
    assert rel_l2(y, ref) < 1e-4
    assert torch.equal(y, yu)


@pytest.mark.parametrize('precision', ['fp32', 'tf32'])
def test_forward_two_lane_split_batch_matches_oracle(dev, precision):
  """``lanes=2``: batches >= 128 are evaluated as two half-batch lanes on two streams (GroupNorm of one lane
  under the other's contractions).  Odd batch -> uneven halves; per-image labels -> the second lane's label offset."""
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision=precision, lanes=2).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  torch.manual_seed(5)
  B = 131
  x = torch.randn(B, 3, 16, 16, device=dev) * 2
  sigma = torch.exp(torch.rand(B, device=dev) * 3 - 2)
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd, cfg, x, sigma)
    y = model(x, sigma)
    y_again = model(x, sigma)
  tol = 1e-4 if precision == 'fp32' else 1e-3
  per_img = ((y - ref).flatten(1).norm(dim=1) / ref.flatten(1).norm(dim=1)).max().item()
  assert per_img < tol, per_img
  assert torch.equal(y, y_again) or precision == 'tf32'   # fp32 path is deterministic; tf32 stats use atomics
  # lane independence: the same images evaluated alone (single lane, B < 128) give the same answer
  with torch.no_grad():
    y_tail = model(x[100:].contiguous(), sigma[100:].contiguous())
  assert rel_l2(y_tail, y[100:]) < (1e-6 if precision == 'fp32' else 2e-4)


def test_state_dict_roundtrip_with_dataparallel_prefix(dev):
  cfg = golden_config('tiny')
  a = seeded_model(cfg, seed=0, precision='fp32').to(dev)
  b = seeded_model(cfg, seed=1, precision='fp32').to(dev)
  x = torch.randn(2, 3, 16, 16, device=dev)
  s = torch.tensor([3.0, 0.5], device=dev)
  ya = a(x, s)
  assert not torch.allclose(ya, b(x, s))
  b.load_state_dict({'module.' + k: v for k, v in a.state_dict().items()})
  assert torch.equal(ya, b(x, s))


def _native_plan(model, sde, predictor, corrector, shape, dev, eps, n_steps=1, snr=0.16):
  from score_sde_pytorch_b200 import native
  plan = native.match_pc_plan(sde=sde, model=model, predictor=predictor, corrector=corrector, shape=shape, snr=snr,
                              n_steps=n_steps, probability_flow=False, continuous=True, eps=eps, device=dev)
  assert plan is not None, 'engine-backed model was not recognised by the native sampler'
  return plan


@pytest.mark.parametrize('combo', ['ve_rd_langevin', 've_em_none', 'vp_rd_langevin', 'vp_em_none'])
def test_native_pc_loop_matches_oracle_same_cuda_seed(dev, combo):
  """Full N-step native loop (CUDA graph + in-kernel Philox) vs the oracle loop drawing torch.randn_like
  on the same CUDA generator seed: identical noise, so trajectories agree to fp32 round-off."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  is_ve = combo.startswith('ve')
  cfg = golden_config('tiny' if is_ve else 'tiny_vp')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (4, 3, 16, 16)
  N = 12 if is_ve else 30
  if is_ve:
    sde, osde, eps = sde_lib.VESDE(0.01, 50, N), SO.VE(0.01, 50, N), 1e-5
  else:
    sde, osde, eps = sde_lib.VPSDE(0.1, 20., N), SO.VP(0.1, 20., N), 1e-3
  pred = sampling.ReverseDiffusionPredictor if '_rd_' in combo else sampling.EulerMaruyamaPredictor
  corr = sampling.LangevinCorrector if combo.endswith('langevin') else sampling.NoneCorrector
  snr = 0.16 if is_ve else 0.01      # the random-init VP model diverges under larger Langevin steps (in the oracle too)
  torch.manual_seed(5)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(77)
  ref, _ = SO.pc_sample(osde, _oracle_model(cfg, sd), shape, 'reverse_diffusion' if '_rd_' in combo else 'euler_maruyama',
                        'langevin' if combo.endswith('langevin') else 'none', snr=snr, n_steps=1, eps=eps,
                        denoise=True, device=dev, x_init=x0)
  assert torch.isfinite(ref).all(), 'oracle trajectory diverged: pick a tamer test configuration'
  off_ref = torch.cuda.default_generators[0].get_offset()
  plan = _native_plan(model, sde, pred, corr, shape, dev, eps, snr=snr)
  torch.cuda.manual_seed(77)
  x, x_mean = plan.run(x0)
  assert torch.cuda.default_generators[0].get_offset() == off_ref     # same generator bookkeeping
  assert rel_l2(x_mean, ref) < 2e-4
  # graph replay == eager launches, and reruns are bit-identical
  plan.use_graph = False
  torch.cuda.manual_seed(77)
  x2, x_mean2 = plan.run(x0)
  plan.use_graph = True
  torch.cuda.manual_seed(77)
  x3, x_mean3 = plan.run(x0)
  assert torch.equal(x_mean, x_mean2) and torch.equal(x, x2)
  assert torch.equal(x_mean, x_mean3) and torch.equal(x, x3)


def test_native_pc_step_with_external_noise_matches_oracle_formulas(dev):
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  om = _oracle_model(cfg, sd)
  shape = (3, 3, 16, 16)
  N = 10
  sde, osde = sde_lib.VESDE(0.01, 50, N), SO.VE(0.01, 50, N)
  plan = _native_plan(model, sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, shape, dev, 1e-5)
  torch.manual_seed(9)
  x = (torch.randn(*shape) * 20).to(dev)
  zc, zp = torch.randn(*shape).to(dev), torch.randn(*shape).to(dev)
  step = 4
  t = torch.ones(shape[0], device=dev) * torch.linspace(1, 1e-5, N, device=dev)[step]
  with torch.no_grad():
    g = osde.score(om, x, t)
    gn = torch.norm(g.reshape(shape[0], -1), dim=-1).mean()
    zn = torch.norm(zc.reshape(shape[0], -1), dim=-1).mean()
    eps_l = (0.16 * zn / gn) ** 2 * 2
    xc = x + eps_l * g + torch.sqrt(eps_l * 2) * zc
    _, G = osde.discretize(xc, t)
    xm = xc + G[:, None, None, None] ** 2 * osde.score(om, xc, t)
    xn = xm + G[:, None, None, None] * zp
  xa, xma = x.clone(), torch.empty_like(x)
  plan.step_external(xa, xma, step, zc, zp)
  assert rel_l2(xma, xm) < 1e-4 and rel_l2(xa, xn) < 1e-4


def test_get_sampling_fn_uses_native_plan_on_cuda(dev):
  from score_sde_pytorch_b200 import sampling, sde_lib, native
  cfg = golden_config('tiny')
  cfg.device = dev
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (2, 3, 16, 16)
  sde = sde_lib.VESDE(0.01, 50, 8)
  fn = sampling.get_sampling_fn(cfg, sde, shape, lambda v: (v + 1.) / 2., 1e-5)
  torch.manual_seed(1); torch.cuda.manual_seed(1)
  s, nfe = fn(model)
  assert nfe == 16 and s.shape == shape and s.is_cuda
  assert getattr(model, '_pc_plans', None), 'native plan was not engaged'
  torch.manual_seed(1); torch.cuda.manual_seed(1)
  ref, _ = SO.pc_sample(SO.VE(0.01, 50, 8), _oracle_model(cfg, sd), shape, eps=1e-5, device=dev)
  assert rel_l2(s, (ref + 1.) / 2.) < 2e-4
  # a user-defined corrector falls back to the generic host loop and still works
  class Half(sampling.Corrector):
    def update_fn(self, x, t):
      return x * 0.5, x * 0.5
  fn2 = sampling.get_pc_sampler(sde, shape, sampling.ReverseDiffusionPredictor, Half, lambda v: v, snr=0.16,
                                continuous=True, eps=1e-5, device=dev)
  s2, _ = fn2(model)
  assert torch.isfinite(s2).all()
