"""`-m gpu`, round-2 additions (VERDICT r01 "Next round" 1b and the advisor's findings):

* VP and sub-VP samplers in BOTH tensor-core operand modes on the CIFAR-10-sized network (round 1 only had them in the
  strict-fp32 mode on the tiny net), and the sub-VP / predictor='none' native loops in fp32 against the oracle;
* single-evaluation parity at batch 256, with persistent multi-tile loops
  and multi-tile GroupNorm sums that batches <= 8 never reach;
* a reference-format checkpoint (module.-prefixed keys, positional EMA shadow list) restored into a fresh model,
  `ema.copy_to`, and the ENGINE's output equals the oracle on the EMA weights ;
* plan/graph validity across batch changes (32 -> 64 -> 32 on one model) and 'cuda' vs 'cuda:0' engine identity.
"""
import pytest
import torch

from helpers import golden_config, seeded_model, rel_l2
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3      # the project's parity bound: per-image relative L2 vs reference <= 1e-3


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _oracle_net(cfg, sd, chunk=64):
  def net(x, labels):
    return torch.cat([NO.ncsnpp_forward(sd, cfg, x[i:i + chunk], labels[i:i + chunk]) for i in range(0, x.shape[0], chunk)])
  return net


def _plan(model, sde, predictor, corrector, shape, dev, eps, snr):
  from score_sde_pytorch_b200 import native
  plan = native.match_pc_plan(sde=sde, model=model, predictor=predictor, corrector=corrector, shape=shape, snr=snr, n_steps=1,
                              probability_flow=False, continuous=True, eps=eps, device=dev)
  assert plan is not None
  return plan


def _vp_cifar_config():
  """The NCSN++ continuous VP / sub-VP CIFAR-10 family (configs/vp/cifar10_ncsnpp_continuous.py:19-59,
  configs/subvp/cifar10_ncsnpp_continuous.py): same network, centred data, no division by sigma."""
  cfg = golden_config('cifar10_ve')
  cfg.model.scale_by_sigma = False
  cfg.data.centered = True
  return cfg


@pytest.mark.parametrize('precision', ['tf32', 'f16'])
@pytest.mark.parametrize('combo', ['vp_rd_langevin', 'vp_em_none', 'subvp_em_none', 'subvp_rd_none'])
def test_vp_subvp_samplers_tensor_core_modes_cifar10(dev, combo, precision):
  """K PC iterations of the (sub-)VP samplers on the 62.8 M-parameter network in tensor-core mode vs the strict-fp32
  oracle, same prior draw, same CUDA noise stream; bound 1e-3 per image."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = _vp_cifar_config()
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape, K, N = (8, 3, 32, 32), 8, 1000
  sub = combo.startswith('subvp')
  sde = (sde_lib.subVPSDE if sub else sde_lib.VPSDE)(0.1, 20., N)
  osde = (SO.SubVP if sub else SO.VP)(0.1, 20., N)
  pred = sampling.ReverseDiffusionPredictor if '_rd_' in combo else sampling.EulerMaruyamaPredictor
  corr = sampling.LangevinCorrector if combo.endswith('langevin') else sampling.NoneCorrector
  snr = 0.01
  torch.manual_seed(3)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(5)
  ref, _ = SO.pc_sample(osde, _oracle_net(cfg, sd), shape, 'reverse_diffusion' if '_rd_' in combo else 'euler_maruyama',
                        'langevin' if combo.endswith('langevin') else 'none', snr=snr, n_steps=1, eps=1e-3, device=dev,
                        x_init=x0, num_iters=K)
  assert torch.isfinite(ref).all()
  plan = _plan(model, sde, pred, corr, shape, dev, 1e-3, snr)
  torch.cuda.manual_seed(5)
  _, xm = plan.run(x0, first_step=0, num_steps=K)
  e = rel_l2(xm, ref)
  print(f'{combo} [{precision}] {K}-step rel-L2 vs oracle: {e:.3e}')
  assert e < TOL_PARITY


@pytest.mark.parametrize('combo', ['ve_none_langevin', 'subvp_em_none', 'subvp_rd_none'])
def test_native_loop_none_predictor_and_subvp_fp32(dev, combo):
  """Strict-fp32 engine on the tiny nets, full N-step loops: predictor='none' returns x (not the Langevin mean) as
  x_mean (sampling.py:241-250; advisor finding r01), and the sub-VP native tables (no GPU test existed)."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  is_ve = combo.startswith('ve')
  cfg = golden_config('tiny' if is_ve else 'tiny_vp')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (4, 3, 16, 16)
  if is_ve:
    N, eps, snr = 12, 1e-5, 0.16
    sde, osde = sde_lib.VESDE(0.01, 50, N), SO.VE(0.01, 50, N)
    pred, corr, opred, ocorr = None, sampling.LangevinCorrector, 'none', 'langevin'
  else:
    N, eps, snr = 30, 1e-3, 0.01
    sde, osde = sde_lib.subVPSDE(0.1, 20., N), SO.SubVP(0.1, 20., N)
    pred = sampling.ReverseDiffusionPredictor if '_rd_' in combo else sampling.EulerMaruyamaPredictor
    corr, opred, ocorr = sampling.NoneCorrector, 'reverse_diffusion' if '_rd_' in combo else 'euler_maruyama', 'none'
  torch.manual_seed(5)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(77)
  ref, _ = SO.pc_sample(osde, _oracle_net(cfg, sd), shape, opred, ocorr, snr=snr, n_steps=1, eps=eps, denoise=True, device=dev, x_init=x0)
  assert torch.isfinite(ref).all()
  plan = _plan(model, sde, pred, corr, shape, dev, eps, snr)
  torch.cuda.manual_seed(77)
  x, x_mean = plan.run(x0)
  assert rel_l2(x_mean, ref) < 2e-4
  if is_ve:
    assert torch.equal(x, x_mean)      # NonePredictor: (x, x)


def test_get_pc_sampler_none_predictor_same_result_native_and_generic(dev):
  """`denoise=True` + predictor=None must not depend on whether the native plan engaged (advisor finding r01)."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('tiny')
  cfg.device = dev
  model = seeded_model(cfg, precision='fp32').to(dev)
  shape = (3, 3, 16, 16)
  sde = sde_lib.VESDE(0.01, 50, 10)
  fn = sampling.get_pc_sampler(sde, shape, None, sampling.LangevinCorrector, lambda v: v, snr=0.16, n_steps=1,
                               continuous=True, denoise=True, eps=1e-5, device=dev)
  torch.manual_seed(2); torch.cuda.manual_seed(2)
  native_s, _ = fn(model)
  assert getattr(model, '_pc_plans', None), 'native plan was not engaged'

  class Same(sampling.LangevinCorrector):   # a user subclass -> generic host loop over the same engine-backed model
    pass
  fn2 = sampling.get_pc_sampler(sde, shape, None, Same, lambda v: v, snr=0.16, n_steps=1, continuous=True, denoise=True,
                                eps=1e-5, device=dev)
  torch.manual_seed(2); torch.cuda.manual_seed(2)
  generic_s, _ = fn2(model)
  assert rel_l2(native_s, generic_s) < 2e-4


@pytest.mark.parametrize('precision', ['tf32', 'f16'])
def test_forward_batch256_plan_matches_small_batch_plan_and_oracle(dev, precision):
  """One evaluation of the headline network at batch 256: every launch is a multi-wave persistent loop and the GroupNorm
  sums of an image come from several tiles/CTAs.
  (a) Kernel-composition check: the same images through batch-8 plans (128-column tiles, one wave) must agree to
  accumulation-order noise - both plans round every operand identically.  (b) Against the strict-fp32 oracle over the
  WHOLE sigma range 0.01..50: a single evaluation carries the 11-bit operand rounding of ~100 chained contractions
  (median ~1e-3 here; cuDNN's own TF32 convolutions are in the same place); the north-star bound of 1e-3 is on the
  SAMPLER output and is held by test_pc_sampler_cifar10_full_1000_steps_within_parity_bound and by bench.py's in-run
  check at batch 1024, so (b) only guards against gross errors."""
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  B = 256
  torch.manual_seed(9)
  sigma = torch.exp(torch.rand(B) * 8.5 - 4.6).to(dev)           # 0.01 .. 50
  x = (torch.randn(B, 3, 32, 32) * (sigma.cpu()[:, None, None, None] + 0.5)).to(dev)
  with torch.no_grad():
    ref = _oracle_net(cfg, sd)(x, sigma)
    y = model(x, sigma).clone()
    y2 = model(x, sigma).clone()
    assert any('[swap-halo]' in n for n in model.op_names())   # the batch-256 plan
    ys = torch.cat([model(x[i:i + 8], sigma[i:i + 8]).clone() for i in range(0, 64, 8)])
  small = ((y[:64] - ys).flatten(1).double().norm(dim=1) / ys.flatten(1).double().norm(dim=1))
  per_img = ((y - ref).flatten(1).double().norm(dim=1) / ref.flatten(1).double().norm(dim=1))
  worst = int(per_img.argmax())
  print(f'batch-256 single eval [{precision}]: vs batch-8 plans max {small.max():.3e}; vs oracle max {per_img.max():.3e} '
        f'(sigma {sigma[worst].item():.3g})  p99 {per_img.quantile(0.99):.3e}  median {per_img.median():.3e}')
  assert small.max().item() < 5e-5
  assert per_img.max().item() < 3e-3 and per_img.median().item() < 1.5e-3
  assert rel_l2(y2, y) < 2e-5          # reruns differ only by the summation order of the fp64 GroupNorm atomics
  # uniform-label fast path (the sampler's case) on the same inputs
  s1 = torch.full((B,), 3.3, device=dev)
  with torch.no_grad():
    assert rel_l2(model(x, s1, labels_uniform=True), model(x, s1)) < 2e-5


@pytest.mark.parametrize('case', ['tiny_fp32', 'cifar10_f16'])
def test_reference_format_checkpoint_ema_weights_drive_the_engine(dev, tmp_path, case):
  """On the GPU: save a checkpoint in the reference's file format (utils.py:7-30: `module.`-prefixed
  model keys, positional EMA shadow list), restore it into a differently-initialised model, `ema.copy_to(...)`
  (run_lib.py:276-284), and the engine - which must repack its device weights - matches the oracle on the EMA weights."""
  from score_sde_pytorch_b200 import utils as butils
  from score_sde_pytorch_b200.models.ema import ExponentialMovingAverage
  name, precision = ('tiny', 'fp32') if case == 'tiny_fp32' else ('cifar10_ve', 'f16')
  cfg = golden_config(name)
  R = cfg.data.image_size
  src = seeded_model(cfg, seed=0, precision=precision).to(dev)
  ema = ExponentialMovingAverage(src.parameters(), decay=0.999)
  with torch.no_grad():                    # two "training steps": the averages now differ from the raw parameters
    for step in range(2):
      for p in src.parameters():
        if p.requires_grad:
          p.add_(torch.randn_like(p) * 0.02 * p.abs().mean())
      ema.update(src.parameters())
  path = str(tmp_path / 'checkpoint_1.pth')
  butils.save_checkpoint(path, dict(optimizer=None, model=src, ema=ema, step=2))
  saved = torch.load(path, map_location='cpu', weights_only=True)
  assert all(k.startswith('module.') for k in saved['model']), 'reference checkpoints carry DataParallel key names'

  dst = seeded_model(cfg, seed=1, precision=precision).to(dev)
  x = torch.randn(2, 3, R, R, device=dev) * 2
  sigma = torch.tensor([4.0, 0.3], device=dev)
  before = dst(x, sigma)                   # builds the engine with the seed-1 weights
  state = dict(optimizer=None, model=dst, ema=ExponentialMovingAverage(dst.parameters(), decay=0.999), step=0)
  state = butils.restore_checkpoint(path, state, device=dev)
  assert state['step'] == 2
  raw = dst(x, sigma)                      # raw (non-averaged) restored weights
  state['ema'].copy_to(dst.parameters())
  y = dst(x, sigma)
  sd_ema = {k: v.detach() for k, v in dst.state_dict().items()}
  for shadow, p in zip(ema.shadow_params, [p for p in dst.parameters() if p.requires_grad]):
    assert torch.equal(shadow.to(dev), p.detach())
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd_ema, cfg, x, sigma)
  tol = 1e-4 if precision == 'fp32' else TOL_PARITY
  assert rel_l2(y, ref) < tol
  assert rel_l2(y, raw) > 10 * tol and rel_l2(raw, before) > 10 * tol, 'the engine kept stale weights'


def test_plans_stay_valid_across_batch_changes(dev):
  """Advisor finding r01 (medium): plan B at batch 32, plan A at batch 64 (the engine reallocates its workspace and
  re-plans), plan B again.  B must re-capture its graph instead of replaying one that points into freed memory."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sde = sde_lib.VESDE(0.01, 50, 6)
  torch.manual_seed(4)
  xa, xb = (torch.randn(64, 3, 16, 16) * 50).to(dev), (torch.randn(32, 3, 16, 16) * 50).to(dev)
  pb = _plan(model, sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, (32, 3, 16, 16), dev, 1e-5, 0.16)
  pa = _plan(model, sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, (64, 3, 16, 16), dev, 1e-5, 0.16)
  assert pa is not pb
  torch.cuda.manual_seed(8); b1 = pb.run(xb)[1]
  torch.cuda.manual_seed(8); a1 = pa.run(xa)[1]
  junk = [torch.randn(1 << 22, device=dev) for _ in range(8)]     # recycle whatever the old workspace occupied
  torch.cuda.manual_seed(8); b2 = pb.run(xb)[1]
  torch.cuda.manual_seed(8); a2 = pa.run(xa)[1]
  del junk
  assert torch.equal(b1, b2) and torch.equal(a1, a2)
  # direct forwards interleaved with plan runs (different batch again) leave the plans usable
  y = model(xb[:5], torch.full((5,), 2.0, device=dev))
  assert torch.isfinite(y).all()
  torch.cuda.manual_seed(8); b3 = pb.run(xb)[1]
  assert torch.equal(b1, b3)


def test_cuda_and_cuda0_name_the_same_engine(dev):
  """Advisor finding r01 (medium): `get_pc_sampler(device='cuda')` followed by `model(x, t)` with x on cuda:0 must not
  destroy and rebuild the engine (torch.device('cuda') != torch.device('cuda:0'))."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sde = sde_lib.VESDE(0.01, 50, 4)
  shape = (2, 3, 16, 16)
  fn = sampling.get_pc_sampler(sde, shape, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, lambda v: v,
                               snr=0.16, n_steps=1, continuous=True, denoise=True, eps=1e-5, device='cuda')
  torch.manual_seed(0); torch.cuda.manual_seed(0)
  s1, _ = fn(model)
  h = model._engine['h'].value
  y = model(torch.randn(2, 3, 16, 16, device=dev), torch.tensor([1.0, 2.0], device=dev))
  assert model._engine['h'].value == h and torch.isfinite(y).all()
  torch.manual_seed(0); torch.cuda.manual_seed(0)
  s2, _ = fn(model)
  assert model._engine['h'].value == h and torch.equal(s1, s2)


@pytest.mark.parametrize('precision', ['f16', 'tf32'])
def test_halo_form_network_equals_nine_load_network_batch256(dev, precision):
  """`halo=True` (default): the swapped-form 3x3 convolutions (128 output channels, 32x32 / 16x16) read three halo copies
  per channel chunk; `halo=False`: one shifted tile per filter tap.  Both add the same products in the same order, so
  they differ only by the order of the fp64 GroupNorm atomics (the level of two runs of one plan).  The plan names say
  which form a launch took."""
  cfg = golden_config('cifar10_ve')
  B = 256
  torch.manual_seed(19)
  sigma = torch.exp(torch.rand(B) * 8.5 - 4.6).to(dev)
  x = (torch.randn(B, 3, 32, 32) * (sigma.cpu()[:, None, None, None] + 0.5)).to(dev)
  ys, names = {}, {}
  for halo in (True, False):
    model = seeded_model(cfg, precision=precision, halo=halo).to(dev)
    with torch.no_grad():
      ys[halo] = model(x, sigma).clone()
    names[halo] = model.op_names()
    del model
  assert any('[swap-halo]' in n for n in names[True])
  assert not any('halo' in n for n in names[False])
  d = ((ys[True] - ys[False]).flatten(1).double().norm(dim=1) / ys[False].flatten(1).double().norm(dim=1))
  print(f'halo=True vs nine-load network [{precision}] batch {B}: max rel-L2 {d.max():.3e}, {sum("halo" in n for n in names[True])} halo launches')
  assert d.max().item() < 2e-5
  model = seeded_model(cfg, precision=precision)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  with torch.no_grad():
    ref = _oracle_net(cfg, sd)(x, sigma)
  for halo in (True,):
    e = ((ys[halo] - ref).flatten(1).double().norm(dim=1) / ref.flatten(1).double().norm(dim=1))
    print(f'halo={halo} vs oracle [{precision}] batch {B}: max {e.max():.3e} median {e.median():.3e}, {sum("halo" in n for n in names[halo])} halo launches')
    assert e.max().item() < 3e-3 and e.median().item() < 1.5e-3


def test_programmatic_dependent_launch_plan_matches_the_serialized_plan(dev):
  """`pdl=True`: every launch of a PC iteration carries the programmatic-dependent-launch attribute and the captured
  graph gets programmatic edges; each kernel still waits for its predecessor's completion (griddepcontrol.wait) before it
  touches memory, so the samples must equal the serialized plan's up to the order of the fp64 GroupNorm atomics - for the
  graph replay and for eager launches - and stay within the parity bound of the oracle."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  cfg = golden_config('cifar10_ve')
  shape = (8, 3, 32, 32)
  sde, osde = sde_lib.VESDE(0.01, 50, 1000), SO.VE(0.01, 50, 1000)
  torch.manual_seed(5)
  x0 = osde.prior_sampling(shape).to(dev)
  outs = {}
  for pdl in (False, True):
    model = seeded_model(cfg, precision='f16', pdl=pdl).to(dev)
    plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.ReverseDiffusionPredictor, corrector=sampling.LangevinCorrector,
                                shape=shape, snr=0.16, n_steps=1, probability_flow=False, continuous=True, eps=1e-5, device=dev)
    for graph in (True, False):
      plan.use_graph = graph
      torch.cuda.manual_seed(77)
      _, xm = plan.run(x0, first_step=0, num_steps=6)
      outs[(pdl, graph)] = xm.clone()
    sd = {k: v.to(dev) for k, v in model.state_dict().items()}
    del plan, model
  base = outs[(False, True)]
  for key, v in outs.items():
    assert torch.isfinite(v).all()
    assert rel_l2(v, base) < 2e-5, f'pdl={key[0]} graph={key[1]} differs from the serialized graph plan'
  torch.cuda.manual_seed(77)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l), shape, eps=1e-5, device=dev, x_init=x0, num_iters=6)
  assert rel_l2(outs[(True, True)], ref) < TOL_PARITY


@pytest.mark.parametrize('combo', ['ve_ancestral_langevin', 've_rd_ald', 've_ancestral_ald', 'vp_ancestral_ald', 'vp_ancestral_none'])
def test_native_loop_ancestral_sampling_and_annealed_langevin(dev, combo):
  """AncestralSamplingPredictor (sampling.py:204-239) and AnnealedLangevinDynamics (:286-319) through the native loop
  (affine tables, the same kernels, in-kernel Philox) against the oracle loop on the same CUDA noise stream - and through
  get_pc_sampler, which must pick the native plan for them."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  is_ve = combo.startswith('ve')
  cfg = golden_config('tiny' if is_ve else 'tiny_vp')
  model = seeded_model(cfg, precision='fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  shape = (4, 3, 16, 16)
  if is_ve:
    sde, osde, eps, snr = sde_lib.VESDE(0.01, 50, 12), SO.VE(0.01, 50, 12), 1e-5, 0.16
  else:
    sde, osde, eps, snr = sde_lib.VPSDE(0.1, 20., 100), SO.VP(0.1, 20., 100), 1e-3, 0.05
  pred_name = 'ancestral_sampling' if 'ancestral' in combo else 'reverse_diffusion'
  corr_name = 'ald' if combo.endswith('ald') else 'langevin' if combo.endswith('langevin') else 'none'
  pred = sampling.AncestralSamplingPredictor if pred_name == 'ancestral_sampling' else sampling.ReverseDiffusionPredictor
  corr = {'ald': sampling.AnnealedLangevinDynamics, 'langevin': sampling.LangevinCorrector, 'none': sampling.NoneCorrector}[corr_name]
  torch.manual_seed(5)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(77)
  ref, _ = SO.pc_sample(osde, _oracle_net(cfg, sd), shape, pred_name, corr_name, snr=snr, n_steps=1, eps=eps, denoise=True, device=dev, x_init=x0)
  assert torch.isfinite(ref).all(), 'oracle trajectory diverged: pick a tamer test configuration'
  off_ref = torch.cuda.default_generators[0].get_offset()
  plan = _plan(model, sde, pred, corr, shape, dev, eps, snr)
  torch.cuda.manual_seed(77)
  x, x_mean = plan.run(x0)
  assert torch.cuda.default_generators[0].get_offset() == off_ref
  e = rel_l2(x_mean, ref)
  print(f'native {combo}: rel-L2 vs oracle loop {e:.2e}')
  assert e < 2e-4
  fn = sampling.get_pc_sampler(sde, shape, pred, corr, lambda v: v, snr=snr, n_steps=1, continuous=True, denoise=True, eps=eps, device=dev)
  torch.manual_seed(5); torch.cuda.manual_seed(77)
  s, _ = fn(model)
  assert getattr(model, '_pc_plans', None), 'native plan was not engaged'
  assert rel_l2(s, ref) < 2e-4


def test_activation_range_report_guards_the_fp16_operand_mode(dev):
  """`precision='f16'` assumes every contraction operand fits IEEE fp16; `activation_range_report` measures the module
  outputs of one evaluation in an fp32-range copy of the network so a checkpoint can be checked first."""
  cfg = golden_config('cifar10_ve')
  model = seeded_model(cfg, precision='f16').to(dev)
  torch.manual_seed(1)
  x = torch.randn(2, 3, 32, 32, device=dev) * 50          # the prior's scale: the largest inputs the sampler sees
  rep = model.activation_range_report(x, torch.tensor([50.0, 0.01], device=dev))
  print(f'activation range: worst module {rep["worst"][0]} max |a| = {rep["worst"][1]:.3g}; {len(rep["max_abs"])} modules')
  assert rep['fits_f16'] and rep['worst'][1] < 6.5e4 and len(rep['max_abs']) > 40
  # a network whose residual stream leaves the fp16 range is reported as such
  with torch.no_grad():
    model.all_modules[3].weight.mul_(1e5)
  model.invalidate_weights()
  assert not model.activation_range_report(x, torch.tensor([50.0, 0.01], device=dev))['fits_f16']
