"""`-m gpu`: the DDPM network (models/ddpm.py; configs/vp/ddpm/cifar10_continuous.py, configs/subvp/cifar10_ddpm_continuous.py,
configs/vp/ddpm/*.py) on the engine - ResnetBlockDDPM with its NIN_0 skip, AttnBlock, Downsample / Upsample with_conv,
32-group GroupNorm, residual scale 1 - against the oracle and against goldens written by the REAL reference
(tools/make_golden_ddpm.py)."""
import pytest
import torch

from ddpm_helpers import golden_config, seeded_ddpm
from helpers import golden, rel_l2
from oracle import ddpm_oracle as DO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3            # bound on SAMPLER outputs
TOL_SINGLE_EVAL_TC = 2.5e-3  # one network evaluation in a tensor-core mode (11-bit operand rounding through the chain)


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def _state(model, dev):
  return {k: v.to(dev) for k, v in model.state_dict().items()}


def test_ddpm_tiny_fp32_matches_oracle_and_reference_golden_per_module(dev):
  g = golden('ddpm_tiny.npz')
  cfg = golden_config('tiny')
  model = seeded_ddpm(cfg, precision='fp32', keep_activations=True).to(dev)
  sd = _state(model, dev)
  x, labels = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = DO.ddpm_forward(sd, cfg, x, labels, taps=taps)
    y = model(x, labels)
  bad, seen = [], 0
  for i in sorted(taps):
    try:
      t = model.tap(i)
    except RuntimeError:
      continue
    seen += 1
    e = rel_l2(t, taps[i])
    if not e < 1e-4:
      bad.append((i, e))
    assert rel_l2(t, torch.from_numpy(g[f'tap{i}']).to(dev)) < 1e-4, f'module {i} vs the reference activation'
  assert not bad, f'diverging modules (index, rel-L2): {bad[:6]}'
  assert seen >= 13      # input conv, every resblock, attention, Downsample and Upsample are recorded
  assert rel_l2(y, ref) < 1e-4
  assert rel_l2(y, torch.from_numpy(g['y']).to(dev)) < 1e-4


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'f16'])
def test_ddpm_cifar10_matches_reference_golden(dev, precision):
  """Full-size DDPM cont. CIFAR-10 network (35.2 M parameters), one evaluation, all three execution modes, against the
  reference's own CPU output; in the tensor-core modes also module by module against the oracle."""
  g = golden('ddpm_cifar10.npz')
  cfg = golden_config('cifar10')
  model = seeded_ddpm(cfg, precision=precision, keep_activations=precision != 'fp32').to(dev)
  sd = _state(model, dev)
  x, labels = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = DO.ddpm_forward(sd, cfg, x, labels, taps=taps)
    y = model(x, labels)
  e_or, e_gold = rel_l2(y, ref), rel_l2(y, torch.from_numpy(g['y']).to(dev))
  print(f'ddpm cifar10 [{precision}] single-eval rel-L2 vs GPU oracle {e_or:.3e}, vs reference CPU golden {e_gold:.3e}')
  if precision == 'fp32':
    assert e_or < 1e-4 and e_gold < 1e-4
    return
  rows = []
  for i in sorted(taps):
    try:
      rows.append((i, rel_l2(model.tap(i), taps[i])))
    except RuntimeError:
      pass
  worst = sorted(rows, key=lambda r: -r[1])[:5]
  print('worst modules', worst)
  assert len(rows) >= 30
  assert all(r[1] < 5e-3 for r in rows), f'worst modules (index, rel-L2): {worst}'
  assert e_or < TOL_SINGLE_EVAL_TC and e_gold < TOL_SINGLE_EVAL_TC
  if precision == 'f16':   # every contraction of the plan runs on fp16 operands, Downsample and NIN_0 inputs included
    names = model.op_names()
    assert any('operand copy' in n for n in names) and any(' s2 ' in n for n in names)


@pytest.mark.parametrize('precision', ['fp32', 'f16'])
@pytest.mark.parametrize('sde_name', ['vp', 'subvp'])
def test_ddpm_sampler_native_loop_matches_oracle(dev, sde_name, precision):
  """The configs' own sampler (Euler-Maruyama predictor, no corrector) through the native PC loop, same prior draw and
  CUDA noise stream as the oracle loop."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  big = precision != 'fp32'
  cfg = golden_config('cifar10' if big else 'tiny')
  model = seeded_ddpm(cfg, precision=precision).to(dev)
  sd = _state(model, dev)
  R = cfg.data.image_size
  shape = (4, 3, R, R)
  N = 12 if big else 20
  sde = sde_lib.VPSDE(0.1, 20., N) if sde_name == 'vp' else sde_lib.subVPSDE(0.1, 20., N)
  osde = SO.VP(0.1, 20., N) if sde_name == 'vp' else SO.SubVP(0.1, 20., N)
  torch.manual_seed(5)
  x0 = osde.prior_sampling(shape).to(dev)
  torch.cuda.manual_seed(77)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, lambda a, l: DO.ddpm_forward(sd, cfg, a, l), shape, 'euler_maruyama', 'none', snr=0.16,
                          n_steps=1, eps=1e-3, denoise=True, device=dev, x_init=x0)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.EulerMaruyamaPredictor, corrector=sampling.NoneCorrector,
                              shape=shape, snr=0.16, n_steps=1, probability_flow=False, continuous=True, eps=1e-3, device=dev)
  assert plan is not None
  torch.cuda.manual_seed(77)
  x, x_mean = plan.run(x0)
  e = rel_l2(x_mean, ref)
  print(f'ddpm {sde_name} EM sampler [{precision}] {N} steps: rel-L2 {e:.3e}')
  assert e < (2e-4 if precision == 'fp32' else TOL_PARITY)


def test_ddpm_discrete_ancestral_host_loop_matches_oracle(dev):
  """configs/vp/ddpm/cifar10.py samples in discrete time (continuous=False, ancestral predictor): get_pc_sampler runs the
  generic host loop over the engine network.  N=20 with beta_max=10 (beta_max=20 makes the last discrete beta 1 at N=20)."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_ddpm(cfg, precision='fp32').to(dev)
  sd = _state(model, dev)
  shape = (3, 3, 16, 16)
  sde, osde = sde_lib.VPSDE(0.1, 10., 20), SO.VP(0.1, 10., 20)
  assert native.match_pc_plan(sde=sde, model=model, predictor=sampling.AncestralSamplingPredictor,
                              corrector=sampling.NoneCorrector, shape=shape, snr=0.16, n_steps=1, probability_flow=False,
                              continuous=False, eps=1e-3, device=dev) is None
  fn = sampling.get_pc_sampler(sde, shape, sampling.AncestralSamplingPredictor, sampling.NoneCorrector, lambda v: v, snr=0.16,
                               n_steps=1, probability_flow=False, continuous=False, denoise=True, eps=1e-3, device=dev)
  torch.manual_seed(31)
  s, nfe = fn(model)
  torch.manual_seed(31)
  ref, nfe_ref = SO.pc_sample(osde, lambda a, l: DO.ddpm_forward(sd, cfg, a, l), shape, 'ancestral_sampling', 'none',
                              snr=0.16, n_steps=1, eps=1e-3, continuous=False, denoise=True, device=dev)
  e = rel_l2(s, ref)
  print(f'ddpm discrete VP ancestral host loop: rel-L2 {e:.3e}, nfe {nfe} / {nfe_ref}')
  assert nfe == nfe_ref and torch.isfinite(s).all()
  assert e < TOL_PARITY


def test_ddpm_device_ode_solver_matches_oracle(dev):
  from score_sde_pytorch_b200 import sampling, sde_lib
  cfg = golden_config('tiny')
  model = seeded_ddpm(cfg, precision='fp32').to(dev)
  sd = _state(model, dev)
  shape = (2, 3, 16, 16)
  sde, osde = sde_lib.VPSDE(0.1, 20., 1000), SO.VP(0.1, 20., 1000)
  torch.manual_seed(61)
  z = sde.prior_sampling(shape).to(dev)
  fn = sampling.get_ode_sampler(sde, shape, lambda v: v, denoise=False, eps=1e-3, device=dev)
  s_dev, nfe_dev = fn(model, z=z.clone())
  assert fn.last_stats['solver'] == 'device'
  s_or, nfe_or = SO.ode_sample(osde, lambda a, l: DO.ddpm_forward(sd, cfg, a, l), shape, z=z.clone(), denoise=False, eps=1e-3,
                               device=dev)
  e = rel_l2(s_dev, s_or)
  print(f'ddpm ode: nfe device {nfe_dev} vs oracle {nfe_or}; rel-L2 {e:.3e}')
  assert abs(nfe_dev - nfe_or) <= 0.05 * nfe_or
  assert e < 1e-3


def test_ddpm_celebahq_256_tf32_matches_oracle(dev):
  """configs/vp/ddpm/celebahq.py (111.6 M parameters, 256x256, 512-channel attention at 16x16 on the separate-launch
  path), one evaluation at batch 1 in tf32."""
  cfg = golden_config('celebahq_256')
  model = seeded_ddpm(cfg, precision='tf32').to(dev)
  sd = _state(model, dev)
  torch.manual_seed(3)
  x = torch.randn(1, 3, 256, 256, device=dev)
  labels = torch.tensor([417.3], device=dev)
  with torch.no_grad():
    y = model(x, labels)
    ref = DO.ddpm_forward(sd, cfg, x, labels)
  e = rel_l2(y, ref)
  print(f'ddpm celebahq-256 [tf32] rel-L2 vs oracle {e:.3e}')
  assert e < TOL_SINGLE_EVAL_TC
  model._release()
