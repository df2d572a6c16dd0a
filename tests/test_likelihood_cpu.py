"""Bits/dim without a GPU: the oracle likelihood and the package's host loop against the fixture the REAL reference wrote
(tests/golden/likelihood_tiny.npz, tools/make_golden_likelihood.py), and the configuration gating of the tangent pass."""
import numpy as np
import pytest
import torch

from ddpm_helpers import seeded_ddpm
from helpers import golden, golden_config, seeded_model, rel_l2
from oracle import ddpm_oracle, likelihood_oracle as LO, ncsnpp_oracle as NO
from oracle import sampling_oracle as SO
from score_sde_pytorch_b200 import configs

SEED = 11   # tools/make_golden_likelihood.py: torch.manual_seed(SEED) right before each likelihood_fn call
NETS = ('tiny_ddpm', 'tiny_ddpmpp')


def net_config(name):
  return configs.tiny_ddpm() if name == 'tiny_ddpm' else golden_config('tiny_ddpmpp')


def oracle_forward(name, cfg):
  """The oracle network with the fixture's weights as a ``model(x, labels)`` callable."""
  if name == 'tiny_ddpm':
    sd = seeded_ddpm(cfg).state_dict()
    return lambda x, l: ddpm_oracle.ddpm_forward(sd, cfg, x, l)
  sd = seeded_model(cfg).state_dict()
  return lambda x, l: NO.ncsnpp_forward(sd, cfg, x, l)


class OracleModule(torch.nn.Module):
  """A plain (autograd-capable) nn.Module around the oracle network: the reference's user-model case."""

  def __init__(self, fwd):
    super().__init__()
    self.fwd = fwd

  def forward(self, x, labels):
    return self.fwd(x, labels)


def inverse_scaler(cfg):
  return (lambda x: (x + 1.) / 2.) if cfg.data.centered else (lambda x: x)


# one CPU run is ~1200 function evaluations with an autograd backward each: a covering subset of the fixture's eight
# (network, SDE, noise) entries; tests/test_gpu_likelihood.py runs the oracle on the others
@pytest.mark.parametrize('name,sde_name,hutch', [('tiny_ddpm', 'vp', 'rademacher'), ('tiny_ddpm', 'subvp', 'gaussian'),
                                                 ('tiny_ddpmpp', 'vp', 'gaussian'), ('tiny_ddpmpp', 'subvp', 'rademacher')])
def test_oracle_likelihood_matches_reference_golden(name, sde_name, hutch):
  g = golden('likelihood_tiny.npz')
  cfg = net_config(name)
  key = f'{name}_{sde_name}_{hutch}'
  sde = SO.VP(0.1, 20., 1000) if sde_name == 'vp' else SO.SubVP(0.1, 20., 1000)
  data, eps = torch.from_numpy(g[f'{name}_data']), torch.from_numpy(g[key + '_eps'])
  bpd, z, nfe = LO.likelihood(sde, oracle_forward(name, cfg), data, eps, inverse_scaler(cfg))
  ref_bpd = g[key + '_bpd']
  assert np.max(np.abs(bpd.numpy() - ref_bpd) / np.abs(ref_bpd)) < 1e-5
  assert rel_l2(z, torch.from_numpy(g[key + '_z'])) < 1e-5
  assert nfe == int(g[key + '_nfe'])


@pytest.mark.parametrize('name', ['tiny_ddpm'])
def test_host_loop_on_plain_module_matches_reference_golden(name):
  """get_likelihood_fn over a plain CPU nn.Module: the reference's autograd host loop, its own Rademacher draw."""
  from score_sde_pytorch_b200 import likelihood, sde_lib
  g = golden('likelihood_tiny.npz')
  cfg = net_config(name)
  key = f'{name}_vp_rademacher'
  model = OracleModule(oracle_forward(name, cfg)).eval()
  fn = likelihood.get_likelihood_fn(sde_lib.VPSDE(0.1, 20., 1000), inverse_scaler(cfg))
  torch.manual_seed(SEED)
  bpd, z, nfe = fn(model, torch.from_numpy(g[f'{name}_data']))
  ref_bpd = g[key + '_bpd']
  assert fn.last_stats['solver'] == 'scipy'
  assert np.max(np.abs(bpd.numpy() - ref_bpd) / np.abs(ref_bpd)) < 1e-5
  assert rel_l2(z, torch.from_numpy(g[key + '_z'])) < 1e-5
  assert nfe == int(g[key + '_nfe'])


def test_host_loop_rk23_runs_on_plain_module():
  from score_sde_pytorch_b200 import likelihood, sde_lib
  g = golden('likelihood_tiny.npz')
  cfg = net_config('tiny_ddpm')
  model = OracleModule(oracle_forward('tiny_ddpm', cfg)).eval()
  fn = likelihood.get_likelihood_fn(sde_lib.subVPSDE(0.1, 20., 1000), inverse_scaler(cfg), hutchinson_type='Gaussian',
                                    method='RK23', rtol=1e-3, atol=1e-3)
  torch.manual_seed(SEED)
  bpd, z, nfe = fn(model, torch.from_numpy(g['tiny_ddpm_data']))
  assert fn.last_stats['solver'] == 'scipy' and nfe > 0
  assert bpd.shape == (2,) and torch.isfinite(bpd).all() and torch.isfinite(z).all()


def test_div_fn_is_the_reference_estimator():
  """get_div_fn on a linear map: eps . (A^T eps) exactly."""
  from score_sde_pytorch_b200 import likelihood
  torch.manual_seed(0)
  A = torch.randn(12, 12, dtype=torch.float64)
  x = torch.randn(3, 1, 3, 4, dtype=torch.float64)
  eps = torch.randn_like(x)
  fn = lambda xx, tt: (xx.reshape(3, 12) @ A.T).reshape(xx.shape)
  div = likelihood.get_div_fn(fn)(x, None, eps)
  e = eps.reshape(3, 12)
  assert torch.allclose(div, ((e @ A) * e).sum(1))


@pytest.mark.parametrize('which', ['fir_ncsnpp', 'progressive', 'f16'])
def test_tangent_gating_rejects_unsupported_configs(which):
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  if which == 'fir_ncsnpp':
    model, field = NCSNpp(configs.tiny_ncsnpp()), 'naive_resample'
  elif which == 'progressive':
    cfg = configs.tiny_progressive(fir=False)
    model, field = NCSNpp(cfg), 'progressive'
  else:
    model, field = NCSNpp(configs.tiny_ddpmpp(), precision='f16'), 'precision'
  with pytest.raises(NotImplementedError, match=field):
    model.check_jvp_supported()


@pytest.mark.parametrize('precision', ['fp32', 'tf32'])
@pytest.mark.parametrize('name', NETS + ('cifar10_ddpm', 'cifar10_ddpmpp'))
def test_tangent_gating_accepts_ddpm_and_ddpmpp(name, precision):
  from score_sde_pytorch_b200.models.ddpm import DDPM
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  cfg = {'tiny_ddpm': configs.tiny_ddpm, 'tiny_ddpmpp': configs.tiny_ddpmpp,
         'cifar10_ddpm': configs.vp_cifar10_ddpm_continuous, 'cifar10_ddpmpp': configs.vp_cifar10_ddpmpp_continuous}[name]()
  model = (DDPM if 'ddpm' in name and 'ddpmpp' not in name else NCSNpp)(cfg, precision=precision)
  model.check_jvp_supported()


def test_jvp_symbols_are_exported():
  from score_sde_pytorch_b200 import _lib
  lib = _lib.load()
  for name in ('b200_ncsnpp_jvp', 'b200_ncsnpp_tap_tangent', 'b200_ode_div_f64'):
    assert hasattr(lib, name)
