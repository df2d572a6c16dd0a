"""`-m gpu`: the DDPM++ family (configs/vp/cifar10_ddpmpp_continuous.py): fir=False naive
2x resampling (up_or_down_sampling.py:59-69), sinusoidal positional embedding (layers.py:515-529, ncsnpp.py:242-247),
no input pyramid, centred data, no division by sigma - through the same engine, against the oracle and against goldens
written by the REAL reference (tools/make_golden_ddpmpp.py)."""
import pytest
import torch

from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO

pytestmark = pytest.mark.gpu
TOL_PARITY = 1e-3          # north-star bound on SAMPLER outputs
TOL_SINGLE_EVAL_TC = 2.5e-3  # one network evaluation in a tensor-core mode: 11-bit operand rounding through ~100 chained
                           # contractions (measured 1.1e-3 tf32 / 1.3e-3 f16 here; the sampler test below holds 1e-3)


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


def test_ddpmpp_tiny_fp32_matches_oracle_and_reference_golden_per_module(dev):
  g = golden('ncsnpp_tiny_ddpmpp.npz')
  cfg = golden_config('tiny_ddpmpp')
  model = seeded_model(cfg, precision='fp32', keep_activations=True).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  x, labels = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd, cfg, x, labels, taps=taps)
    y = model(x, labels)
  bad = []
  for i in sorted(taps):
    try:
      e = rel_l2(model.tap(i), taps[i])
    except RuntimeError:
      continue
    if not e < 1e-4:
      bad.append((i, e))
    key = f'tap{i}'
    if key in g and taps[i].dim() == 4:
      assert rel_l2(model.tap(i), torch.from_numpy(g[key]).to(dev)) < 1e-4, f'module {i} vs the reference activation'
  assert not bad, f'diverging modules (index, rel-L2): {bad[:6]}'
  assert rel_l2(y, ref) < 1e-4
  assert rel_l2(y, torch.from_numpy(g['y']).to(dev)) < 1e-4


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'f16'])
def test_ddpmpp_cifar10_matches_reference_golden(dev, precision):
  """Full-size DDPM++ cont. (VP) CIFAR-10 network, one evaluation, all three execution modes, against the reference's
  own CPU output; in the tensor-core modes also module by module against the oracle."""
  g = golden('ncsnpp_cifar10_ddpmpp.npz')
  cfg = golden_config('cifar10_ddpmpp')
  model = seeded_model(cfg, precision=precision, keep_activations=precision != 'fp32').to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  x, labels = torch.from_numpy(g['x']).to(dev), torch.from_numpy(g['sigma']).to(dev)
  taps = {}
  with torch.no_grad():
    ref = NO.ncsnpp_forward(sd, cfg, x, labels, taps=taps)
    y = model(x, labels)
  e_or, e_gold = rel_l2(y, ref), rel_l2(y, torch.from_numpy(g['y']).to(dev))
  print(f'ddpm++ cifar10 [{precision}] single-eval rel-L2 vs GPU oracle {e_or:.3e}, vs reference CPU golden {e_gold:.3e}')
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
  assert all(r[1] < 5e-3 for r in rows), f'worst modules (index, rel-L2): {worst}'
  assert e_or < TOL_SINGLE_EVAL_TC and e_gold < TOL_SINGLE_EVAL_TC


@pytest.mark.parametrize('precision', ['fp32', 'f16'])
@pytest.mark.parametrize('sde_name', ['vp', 'subvp'])
def test_ddpmpp_sampler_native_loop_matches_oracle(dev, sde_name, precision):
  """The config's own sampler (Euler-Maruyama predictor, no corrector; configs/vp/cifar10_ddpmpp_continuous.py:33-35)
  through get_pc_sampler -> native plan, K steps, same prior draw and CUDA noise stream as the oracle loop."""
  from score_sde_pytorch_b200 import native, sampling, sde_lib
  big = precision != 'fp32'
  cfg = golden_config('cifar10_ddpmpp' if big else 'tiny_ddpmpp')
  model = seeded_model(cfg, precision=precision).to(dev)
  sd = {k: v.to(dev) for k, v in model.state_dict().items()}
  R = cfg.data.image_size
  shape = (4, 3, R, R)
  N = 12 if big else 20
  sde = sde_lib.VPSDE(0.1, 20., N) if sde_name == 'vp' else sde_lib.subVPSDE(0.1, 20., N)
  osde = SO.VP(0.1, 20., N) if sde_name == 'vp' else SO.SubVP(0.1, 20., N)
  torch.manual_seed(5)
  x0 = osde.prior_sampling(shape).to(dev)
  net = lambda a, l: NO.ncsnpp_forward(sd, cfg, a, l)
  torch.cuda.manual_seed(77)
  with torch.no_grad():
    ref, _ = SO.pc_sample(osde, net, shape, 'euler_maruyama', 'none', snr=0.16, n_steps=1, eps=1e-3, denoise=True, device=dev, x_init=x0)
  plan = native.match_pc_plan(sde=sde, model=model, predictor=sampling.EulerMaruyamaPredictor, corrector=sampling.NoneCorrector,
                              shape=shape, snr=0.16, n_steps=1, probability_flow=False, continuous=True, eps=1e-3, device=dev)
  assert plan is not None
  torch.cuda.manual_seed(77)
  x, x_mean = plan.run(x0)
  e = rel_l2(x_mean, ref)
  print(f'ddpm++ {sde_name} EM sampler [{precision}] {N} steps: rel-L2 {e:.3e}')
  assert e < (2e-4 if precision == 'fp32' else TOL_PARITY)
