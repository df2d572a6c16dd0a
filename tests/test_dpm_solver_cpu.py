"""CPU: the multistep DPM-Solver / DPM-Solver++ sampler (`sampling.method = 'dpm_solver'`) - its log-SNR schedules, the
convergence of its tables on an analytic score, the tables against the float64 oracle, the host loop against the oracle
loop on the tiny networks, dispatch, refusals and the C ABI fields of the native loop."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import golden_config, rel_l2, seeded_model
from oracle import dpm_solver_oracle as DO, ncsnpp_oracle as NO
from score_sde_pytorch_b200 import _lib, configs, native, sampling, sde_lib

SDES = {'ve': lambda: sde_lib.VESDE(0.01, 50., 1000), 'vp': lambda: sde_lib.VPSDE(0.1, 20., 1000),
        'subvp': lambda: sde_lib.subVPSDE(0.1, 20., 1000)}
ALGORITHMS = ('dpmsolver++', 'dpmsolver')
MU, S2 = 0.7, 0.25   # the analytic data distribution N(MU, S2 I)


def oracle_marginal(kind):
  return DO.Marginal(kind)


def ab(sde, t):
  la, ls, _ = native.marginal_schedule(sde)
  return np.exp(la(t)), np.exp(ls(t))


class GaussianScore(torch.nn.Module):
  """Exact score of N(MU, S2 I) data under the SDE, returned in the SDE's get_score_fn convention: the score itself for VE
  (label sigma_t), -sigma_t * score for (sub-)VP (label 999 t)."""

  def __init__(self, sde):
    super().__init__()
    self.sde = sde

  def forward(self, x, labels):
    sde = self.sde
    if isinstance(sde, sde_lib.VESDE):
      t = torch.log(labels / sde.sigma_min) / np.log(sde.sigma_max / sde.sigma_min)
    else:
      t = labels / 999
    mean_coef, std = sde.marginal_prob(torch.ones_like(x), t)
    a = mean_coef[:, :1, :1, :1]
    s = std[:, None, None, None]
    score = -(x - a * MU) / (a * a * S2 + s * s)
    return score if isinstance(sde, sde_lib.VESDE) else -s * score


def exact_solution(sde, t, xT):
  a, s = ab(sde, t)
  aT, sT = ab(sde, float(sde.T))
  return a * MU + np.sqrt((a * a * S2 + s * s) / (aT * aT * S2 + sT * sT)) * (xT - aT * MU)


def analytic_score(sde, x, t):
  a, s = ab(sde, t)
  return -(x - a * MU) / (a * a * S2 + s * s)


@pytest.mark.parametrize('kind', list(SDES))
def test_schedule_matches_marginal_prob_and_inverts(kind):
  sde = SDES[kind]()
  la, ls, t_of_lambda = native.marginal_schedule(sde)
  t = np.linspace(1e-5, 1., 2001)
  mean, std = sde.marginal_prob(torch.ones(t.size, dtype=torch.float64), torch.from_numpy(t))
  np.testing.assert_allclose(np.exp(la(t)), mean.numpy(), rtol=1e-13)
  # sde.marginal_prob's 1 - exp(2 log alpha) cancels near t = 0 (the schedule uses expm1), hence the looser bound
  np.testing.assert_allclose(np.exp(ls(t)), std.numpy(), rtol=1e-9)
  lam = la(t) - ls(t)
  assert np.all(np.diff(lam) < 0)
  assert np.max(np.abs(t_of_lambda(lam) - t)) < 1e-12
  mg = oracle_marginal(kind)
  np.testing.assert_allclose(lam, mg.lam(torch.from_numpy(t)).numpy(), rtol=1e-11, atol=1e-12)


def one_step_error(sde, algorithm, order, h, t_mid=0.5):
  """|x_{i+1} - x(lambda_i + h)| for a step at order `order` from t_mid with exact history at equal lambda spacing h."""
  la, ls, t_of_lambda = native.marginal_schedule(sde)
  l0 = la(t_mid) - ls(t_mid)
  t = t_of_lambda(l0 + h * np.arange(-order + 1, 2))
  tab = native.multistep_coefficients(sde, t, list(range(1, order + 1)), algorithm)
  xT = 1.3 * ab(sde, 1.)[1]
  xs = exact_solution(sde, t, xT)
  m = [tab['mq'][j] * xs[j] + tab['ms'][j] * analytic_score(sde, xs[j], t[j]) for j in range(order)]
  i = order - 1
  xn = tab['pa'][i] * xs[i] + tab['pb'][i] * m[i]
  if order > 1:
    xn += tab['pm1'][i] * m[i - 1]
  if order > 2:
    xn += tab['pm2'][i] * m[i - 2]
  return abs(xn - xs[-1])


@pytest.mark.parametrize('kind', list(SDES))
@pytest.mark.parametrize('algorithm', ALGORITHMS)
@pytest.mark.parametrize('order', [1, 2, 3])
def test_local_error_is_of_order_plus_one(kind, algorithm, order):
  sde = SDES[kind]()
  hs = np.array([0.4, 0.2, 0.1, 0.05, 0.025])
  errs = np.array([one_step_error(sde, algorithm, order, h) for h in hs])
  slope = np.polyfit(np.log(hs), np.log(errs), 1)[0]
  assert abs(slope - (order + 1)) < 0.3, (slope, errs)


@pytest.mark.parametrize('kind', list(SDES))
@pytest.mark.parametrize('algorithm', ALGORITHMS)
@pytest.mark.parametrize('order', [1, 2, 3])
def test_global_error_converges_at_the_order(kind, algorithm, order):
  """The sampler's host loop in float64 on the analytic score: from 20 steps on, the final-state error halves (order 1)
  or quarters (orders 2 and 3) at least with each doubling of the steps.  (From 10 to 20 steps, where a step spans more
  than one unit of log-SNR, order 2 is not yet in its asymptotic range: there the error only has to drop.)"""
  sde = SDES[kind]()
  eps = 1e-3
  torch.manual_seed(0)
  xT = torch.randn(2, 1, 2, 2, dtype=torch.float64) * ab(sde, 1.)[1]
  want = torch.from_numpy(exact_solution(sde, eps, xT.numpy()))
  errs = []
  for steps in (10, 20, 40, 80):
    fn = sampling.get_dpm_solver_sampler(sde, tuple(xT.shape), lambda v: v, steps=steps, order=order, algorithm=algorithm,
                                         eps=eps, device='cpu')
    x, nfe = fn(GaussianScore(sde), z=xT.clone())
    assert nfe == steps and x.dtype == torch.float64 and fn.last_stats['loop'] == 'host'
    errs.append((x - want).abs().max().item())
  p = 1 if order == 1 else 2
  ratios = [errs[j] / errs[j + 1] for j in range(3)]
  assert ratios[0] > 1.5 and all(r >= 2 ** p * 0.8 for r in ratios[1:]), (errs, ratios)


CASES = [('ve', 10, 3, 'logSNR'), ('vp', 10, 3, 'logSNR'), ('subvp', 10, 3, 'logSNR'), ('vp', 7, 3, 'time_uniform'),
         ('ve', 5, 2, 'time_quadratic'), ('subvp', 20, 2, 'logSNR'), ('vp', 3, 1, 'logSNR'), ('ve', 50, 3, 'time_uniform'),
         ('subvp', 1, 3, 'logSNR')]


@pytest.mark.parametrize('kind,steps,order,skip_type', CASES)
@pytest.mark.parametrize('algorithm', ALGORITHMS)
def test_tables_equal_the_oracle(kind, steps, order, skip_type, algorithm):
  sde = SDES[kind]()
  tab = native.build_multistep_tables(sde, steps, order, algorithm, skip_type, 1e-3)
  ref = DO.coefficients(oracle_marginal(kind), steps, order, algorithm, skip_type, eps=1e-3)
  np.testing.assert_allclose(tab['t'], ref['t'].numpy(), rtol=1e-12, atol=0)
  assert list(tab['orders']) == DO.step_orders(steps, order)
  for k in ('pa', 'pb', 'pm1', 'pm2', 'mq', 'ms'):
    scale = np.abs(ref[k].numpy()).max() + 1e-300
    assert np.abs(tab[k] - ref[k].numpy()).max() <= 1e-12 * scale, k
  assert tab['label'].dtype == np.float32 and tab['label'].shape == (steps,)


def test_step_orders_warm_up_and_short_schedules():
  assert native.multistep_orders(5, 3) == [1, 2, 3, 2, 1]
  assert native.multistep_orders(9, 3) == [1, 2, 3, 3, 3, 3, 3, 2, 1]
  assert native.multistep_orders(10, 3) == [1, 2] + [3] * 8
  assert native.multistep_orders(20, 2) == [1] + [2] * 19
  assert native.multistep_orders(1, 3) == [1]


@pytest.mark.parametrize('kind', list(SDES))
@pytest.mark.parametrize('algorithm', ALGORITHMS)
def test_order_one_is_ddim(kind, algorithm):
  """x_t = alpha_t x0 + sigma_t eps with eps = -sigma_s score, x0 = (x_s - sigma_s eps) / alpha_s."""
  sde = SDES[kind]()
  tab = native.build_multistep_tables(sde, 12, 1, algorithm, 'logSNR', 1e-3)
  x, score = 0.37, -1.9
  for i in range(12):
    a_s, s_s = ab(sde, tab['t'][i])
    a_t, s_t = ab(sde, tab['t'][i + 1])
    e = -s_s * score
    want = a_t * (x - s_s * e) / a_s + s_t * e
    m = tab['mq'][i] * x + tab['ms'][i] * score
    got = tab['pa'][i] * x + tab['pb'][i] * m
    assert tab['pm1'][i] == 0 and tab['pm2'][i] == 0
    assert abs(got - want) <= 1e-12 * max(1., abs(want)), (i, got, want)


class OracleNet(torch.nn.Module):
  """A plain module over the oracle network arithmetic (fp32), with the goldens' weights."""

  def __init__(self, cfg):
    super().__init__()
    self.cfg = cfg
    self.sd = seeded_model(cfg).state_dict()

  def forward(self, x, labels):
    return NO.ncsnpp_forward(self.sd, self.cfg, x.float(), labels.float())


def oracle_score(kind, net, sde):
  mg = oracle_marginal(kind)

  def score(x, t):
    if kind == 've':
      return net(x, mg.sigma(t)).double()
    return -net(x, t * 999).double() / mg.sigma(t)[:, None, None, None]
  return score


@pytest.mark.parametrize('kind,name', [('ve', 'tiny'), ('vp', 'tiny_ddpmpp'), ('subvp', 'tiny_ddpmpp')])
@pytest.mark.parametrize('algorithm', ALGORITHMS)
@pytest.mark.parametrize('order', [2, 3])
def test_host_loop_matches_oracle_loop_on_tiny_networks(kind, name, algorithm, order):
  cfg = golden_config(name)
  net = OracleNet(cfg)
  sde = SDES[kind]()
  shape = (2, cfg.data.num_channels, cfg.data.image_size, cfg.data.image_size)
  torch.manual_seed(3)
  z = sde.prior_sampling(shape)
  fn = sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, steps=10, order=order, algorithm=algorithm, device='cpu')
  with torch.no_grad():
    x, nfe = fn(net, z=z.clone())
    ref = DO.sample(oracle_marginal(kind), oracle_score(kind, net, sde), z.double(), 10, order, algorithm)
  err = rel_l2(x, ref)
  print(f'{kind} {algorithm} order {order}: host loop (fp32) vs oracle loop (fp64 state) rel-L2 {err:.2e}')
  assert x.dtype == torch.float32 and nfe == 10 and fn.last_stats == dict(loop='host', steps=10, order=order, nfe=10)
  assert err < 2e-5


def test_get_sampling_fn_dispatch_and_defaults():
  cfg = configs.ve_cifar10_ncsnpp_continuous()
  cfg.device = torch.device('cpu')
  cfg.sampling.method = 'dpm_solver'
  cfg.sampling.noise_removal = False
  sde = sde_lib.VESDE(0.01, 50., 1000)
  shape = (1, 1, 2, 2)
  fn = sampling.get_sampling_fn(cfg, sde, shape, lambda v: v, 1e-3)
  x, nfe = fn(GaussianScore(sde), z=torch.randn(shape, dtype=torch.float64) * 50)
  assert nfe == 20 and fn.last_stats == dict(loop='host', steps=20, order=3, nfe=20)
  cfg.sampling.update(dpm_steps=12, dpm_order=2, dpm_algorithm='dpmsolver', dpm_skip_type='time_uniform', noise_removal=True)
  fn = sampling.get_sampling_fn(cfg, sde, shape, lambda v: v, 1e-3)
  z = torch.randn(shape, dtype=torch.float64) * 50
  x2, nfe = fn(GaussianScore(sde), z=z.clone())
  assert nfe == 13 and fn.last_stats == dict(loop='host', steps=12, order=2, nfe=13)
  # the same 12 steps without noise_removal, then get_ode_sampler's denoising step
  plain = sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, steps=12, order=2, algorithm='dpmsolver',
                                          skip_type='time_uniform', eps=1e-3, device='cpu')
  x1, _ = plain(GaussianScore(sde), z=z.clone())
  assert torch.equal(x2, sampling._denoise_update(sde, GaussianScore(sde), x1, 1e-3))
  cfg.sampling.method = 'nope'
  with pytest.raises(ValueError):
    sampling.get_sampling_fn(cfg, sde, shape, lambda v: v, 1e-3)


def test_refusals():
  sde = sde_lib.VPSDE(0.1, 20., 1000)
  shape = (1, 3, 4, 4)
  for kw in (dict(order=4), dict(order=0), dict(steps=0), dict(algorithm='unipc'), dict(skip_type='karras')):
    with pytest.raises(ValueError):
      sampling.get_dpm_solver_sampler(sde, shape, lambda v: v, device='cpu', **kw)

  class OtherSDE(sde_lib.VPSDE):
    pass
  with pytest.raises(NotImplementedError, match='OtherSDE'):
    sampling.get_dpm_solver_sampler(OtherSDE(), shape, lambda v: v, device='cpu')

  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2
  cfg = configs.tiny_ncsnv2()
  net = NCSNv2(cfg)
  fn = sampling.get_dpm_solver_sampler(sde_lib.VESDE(0.01, 50., 1000), (1, cfg.data.num_channels, cfg.data.image_size,
                                                                          cfg.data.image_size), lambda v: v, device='cpu')
  with pytest.raises(NotImplementedError, match='noise-level indices'):
    fn(net)


def test_pc_config_multistep_fields_trail_the_struct():
  assert [f[0] for f in _lib.PcConfig._fields_][-5:] == ['noise_nhwc', 'mq', 'mr', 'pm1', 'pm2']
  off = _lib.PcConfig.noise_nhwc.offset
  ptr = ctypes.sizeof(ctypes.c_void_p)
  assert _lib.PcConfig.mq.offset > off and _lib.PcConfig.mq.offset % ptr == 0
  assert [getattr(_lib.PcConfig, k).offset - _lib.PcConfig.mq.offset for k in ('mr', 'pm1', 'pm2')] == [ptr, 2 * ptr, 3 * ptr]
  assert ctypes.sizeof(_lib.PcConfig) == _lib.PcConfig.pm2.offset + ptr
  cfg = _lib.PcConfig()
  assert not cfg.mq and not cfg.mr and not cfg.pm1 and not cfg.pm2
