"""`-m gpu`: the device-resident ODE solve with scipy's RK23 and DOP853 (score_sde_pytorch_b200/ode.py + csrc/ode.cu),
for the probability-flow sampler and for bits/dim, held to
  * scipy itself over the same engine network and right-hand side (`device_solver=False`): the controller is scipy's, the
    stage sums differ only in float64 rounding, so the evaluation counts agree exactly and the samples to 1e-12;
  * the fixture the REAL reference wrote on CPU (tests/golden/ode_methods_tiny.npz, tools/make_golden_ode_methods.py);
  * itself: the DOP853 error reduction is deterministic, and RK45 keeps the evaluation counts and bits it had."""
import ctypes

import numpy as np
import pytest
import torch

from ddpm_helpers import seeded_ddpm
from helpers import golden, golden_config, rel_l2, seeded_model

pytestmark = pytest.mark.gpu
METHODS = ('RK23', 'DOP853')


@pytest.fixture(scope='module')
def dev():
  import gpu_util
  gpu_util.strict_fp32()
  return torch.device('cuda:0')


@pytest.fixture(scope='module')
def nets(dev):
  """The fixture networks with the goldens' weights, fp32, built once per module."""
  from score_sde_pytorch_b200 import configs
  cache = {}

  def get(name):
    if name not in cache:
      if name == 'tiny':
        model = seeded_model(golden_config('tiny'), precision='fp32')
      elif name == 'tiny_ddpm':
        model = seeded_ddpm(configs.tiny_ddpm(), precision='fp32')
      else:
        model = seeded_model(configs.tiny_ddpmpp(), precision='fp32')
      cache[name] = model.to(dev)
    return cache[name]

  return get


@pytest.fixture(scope='module')
def fixture():
  return golden('ode_methods_tiny.npz')


def sampler_case(case):
  """case -> (network, SDE, eps): tools/make_golden_ode_methods.py."""
  from score_sde_pytorch_b200 import sde_lib
  return {'ve': ('tiny', sde_lib.VESDE(0.01, 50, 1000), 1e-5),
          'vp_ddpm': ('tiny_ddpm', sde_lib.VPSDE(0.1, 20., 1000), 1e-3),
          'vp_ddpmpp': ('tiny_ddpmpp', sde_lib.VPSDE(0.1, 20., 1000), 1e-3)}[case]


def inverse_scaler(name):
  from score_sde_pytorch_b200 import configs
  centered = (configs.tiny_ddpm() if name == 'tiny_ddpm' else configs.tiny_ddpmpp()).data.centered
  return (lambda v: (v + 1.) / 2.) if centered else (lambda v: v)


@pytest.mark.parametrize('case', ['ve', 'vp_ddpm', 'vp_ddpmpp'])
@pytest.mark.parametrize('method', METHODS)
def test_device_sampler_matches_scipy_and_reference(dev, nets, fixture, method, case):
  from score_sde_pytorch_b200 import ode, sampling
  name, sde, eps = sampler_case(case)
  model = nets(name)
  z = torch.from_numpy(fixture[case + '_z']).to(dev)
  shape = tuple(z.shape)
  fn_dev = sampling.get_ode_sampler(sde, shape, lambda v: v, eps=eps, method=method, device=dev)
  fn_host = sampling.get_ode_sampler(sde, shape, lambda v: v, eps=eps, method=method, device=dev, device_solver=False)
  s_dev, nfe_dev = fn_dev(model, z=z.clone())
  s_host, nfe_host = fn_host(model, z=z.clone())
  stats = fn_dev.last_stats
  e_host = rel_l2(s_dev, s_host)
  e_ref = rel_l2(s_dev, torch.from_numpy(fixture[f'{method}_{case}']).to(dev))
  nfe_ref = int(fixture[f'{method}_{case}_nfe'])
  print(f'{method} sampler [{case}]: nfe device {nfe_dev}, scipy {nfe_host}, reference (CPU) {nfe_ref}; '
        f'rel-L2 vs scipy {e_host:.2e}, vs reference {e_ref:.2e}; host reads {stats["host_scalar_reads"]}')
  assert stats['solver'] == 'device' and stats['method'] == method
  assert fn_host.last_stats == dict(nfev=nfe_host, solver='scipy', method=method)
  assert nfe_dev == nfe_host
  assert e_host <= 1e-12
  # one transfer per attempted step (n_stages evaluations each after the first two), plus select_initial_step's norms
  assert stats['host_scalar_reads'] == (nfe_dev - 2) // ode.METHODS[method].n_stages + 3
  # the reference ran in float32 on CPU: a different network arithmetic that the adaptive steps follow, the bound of the
  # RK45 sampler's test (tests/test_gpu_ode.py; measured on an H100: <= 1.4e-5 here, DOP853 on VE the largest, and the
  # evaluation counts equal the reference's or within 1 %)
  assert e_ref < 1e-2


@pytest.mark.parametrize('name', ['tiny_ddpm', 'tiny_ddpmpp'])
@pytest.mark.parametrize('method', METHODS)
def test_device_likelihood_matches_host_loop(dev, nets, fixture, method, name):
  """rtol = atol = 1e-3: the host loop runs scipy over the same engine JVP and the same float64 divergence products."""
  from score_sde_pytorch_b200 import likelihood, sde_lib
  model = nets(name)
  key = f'{method}_lik_{name}'
  data = torch.from_numpy(fixture[f'{name}_data']).to(dev)
  eps = torch.from_numpy(fixture[key + '_eps']).to(dev)
  sde = sde_lib.VPSDE(0.1, 20., 1000)
  fn = likelihood.get_likelihood_fn(sde, inverse_scaler(name), rtol=1e-3, atol=1e-3, method=method)
  fn_host = likelihood.get_likelihood_fn(sde, inverse_scaler(name), rtol=1e-3, atol=1e-3, method=method, device_solver=False)
  bpd, z, nfe = fn(model, data, epsilon=eps)
  hbpd, hz, hnfe = fn_host(model, data, epsilon=eps)
  e = ((bpd - hbpd).abs() / hbpd.abs()).max().item()
  print(f'{key} rtol=1e-3: bpd {bpd.tolist()} host {hbpd.tolist()}; nfe {nfe} / {hnfe}; bpd rel {e:.2e}, '
        f'z rel-L2 {rel_l2(z, hz):.2e}')
  assert fn.last_stats['solver'] == 'device' and fn.last_stats['method'] == method
  assert fn_host.last_stats['solver'] == 'scipy'
  assert nfe == hnfe and e < 1e-4


@pytest.mark.parametrize('name', ['tiny_ddpm', 'tiny_ddpmpp'])
@pytest.mark.parametrize('method', METHODS)
def test_device_likelihood_matches_reference_golden(dev, nets, fixture, method, name):
  """The reference's default tolerances (rtol = atol = 1e-5) and its own Hutchinson draw."""
  from score_sde_pytorch_b200 import likelihood, sde_lib
  model = nets(name)
  key = f'{method}_lik_{name}'
  data = torch.from_numpy(fixture[f'{name}_data']).to(dev)
  eps = torch.from_numpy(fixture[key + '_eps']).to(dev)
  fn = likelihood.get_likelihood_fn(sde_lib.VPSDE(0.1, 20., 1000), inverse_scaler(name), method=method)
  bpd, z, nfe = fn(model, data, epsilon=eps)
  ref_bpd = fixture[key + '_bpd']
  e = float(np.max(np.abs(bpd.cpu().numpy() - ref_bpd) / np.abs(ref_bpd)))
  print(f'{key}: bpd {bpd.tolist()} reference {ref_bpd.tolist()}; nfe {nfe} / {int(fixture[key + "_nfe"])}; '
        f'bpd rel {e:.2e}')
  assert fn.last_stats['solver'] == 'device' and fn.last_stats['method'] == method
  # the reference ran in float32 on CPU: the random-weight networks make the likelihood ODE stiff (2600-3300
  # evaluations), and over its trajectory the float32 GPU and CPU right-hand sides drift apart.  RK45 on the same
  # networks reaches 8.2e-3 (tests/test_gpu_likelihood.py); measured here on an H100: <= 2.4e-4, evaluation counts within 2 %
  assert e < 1e-2


def _sumsq2(ws, y, y_new, K, e5, e3):
  from score_sde_pytorch_b200 import _lib
  arr = lambda c: (ctypes.c_double * 16)(*c)
  _lib.call('b200_ode_error_sumsq2_f64', _lib.ptr(y), _lib.ptr(y_new), _lib.ptr(K), y.numel(), arr(e5), arr(e3), len(e5),
            1e-5, 1e-5, _lib.ptr(ws), _lib.stream_ptr(y.device))
  return ws[:2].clone()


def test_dop853_error_reduction_is_deterministic_and_exact(dev):
  """Two runs give the same bits; each sum equals b200_ode_error_sumsq_f64's (h = 1) bit for bit, and float64 torch to
  round-off.  n spans the full 1024-block grid with several elements per thread."""
  from score_sde_pytorch_b200 import _lib, ode
  g = torch.Generator(device=dev).manual_seed(3)
  n = 3 * 1024 * 1024 + 1037
  K = torch.randn(ode.DOP853.n_stages + 1, n, generator=g, device=dev, dtype=torch.float64)
  y = torch.randn(n, generator=g, device=dev, dtype=torch.float64)
  y_new = y + 1e-3 * torch.randn(n, generator=g, device=dev, dtype=torch.float64)
  ws = torch.zeros(int(_lib.load().b200_ode_workspace_doubles()), dtype=torch.float64, device=dev)
  e5, e3 = ode.DOP853.E5, ode.DOP853.E3
  a = _sumsq2(ws, y, y_new, K, e5, e3)
  b = _sumsq2(ws, y, y_new, K, e5, e3)
  assert torch.equal(a, b)
  for i, e in enumerate((e5, e3)):
    _lib.call('b200_ode_error_sumsq_f64', _lib.ptr(y), _lib.ptr(y_new), _lib.ptr(K), n, (ctypes.c_double * 16)(*e), len(e),
              1.0, 1e-5, 1e-5, _lib.ptr(ws), _lib.stream_ptr(dev))
    assert ws[0].item() == a[i].item()
    scale = 1e-5 + torch.maximum(y.abs(), y_new.abs()) * 1e-5
    ref = ((torch.tensor(e, dtype=torch.float64, device=dev) @ K / scale) ** 2).sum().item()
    assert abs(a[i].item() - ref) <= 1e-12 * ref


def test_dop853_solve_is_deterministic(dev, nets, fixture):
  from score_sde_pytorch_b200 import likelihood, sde_lib
  model = nets('tiny_ddpm')
  data = torch.from_numpy(fixture['tiny_ddpm_data']).to(dev)
  eps = torch.from_numpy(fixture['DOP853_lik_tiny_ddpm_eps']).to(dev)
  fn = likelihood.get_likelihood_fn(sde_lib.VPSDE(0.1, 20., 1000), inverse_scaler('tiny_ddpm'), rtol=1e-3, atol=1e-3,
                                    method='DOP853')
  a = fn(model, data, epsilon=eps)
  b = fn(model, data, epsilon=eps)
  assert a[2] == b[2] and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize('case,nfev', [('ve', 410), ('vp', 488), ('subvp', 476)])
def test_rk45_keeps_its_evaluation_counts_and_bits(dev, case, nfev):
  """The RK45 sampler on the tests/golden/ode_tiny.npz cases: the evaluation counts this solver had before it took other
  methods, and the same bits as scipy's own RK45 over the same network."""
  from score_sde_pytorch_b200 import sampling, sde_lib
  g = golden('ode_tiny.npz')
  name, sde, eps, denoise = {'ve': ('tiny', sde_lib.VESDE(0.01, 50, 1000), 1e-5, False),
                             'vp': ('tiny_ddpmpp', sde_lib.VPSDE(0.1, 20., 1000), 1e-3, False),
                             'subvp': ('tiny_ddpmpp', sde_lib.subVPSDE(0.1, 20., 1000), 1e-3, True)}[case]
  model = seeded_model(golden_config(name), precision='fp32').to(dev)
  z = torch.from_numpy(g[case + '_z']).to(dev)
  shape = tuple(z.shape)
  fn = sampling.get_ode_sampler(sde, shape, lambda v: v, denoise=denoise, eps=eps, device=dev)
  fn_host = sampling.get_ode_sampler(sde, shape, lambda v: v, denoise=denoise, eps=eps, device=dev, device_solver=False)
  torch.manual_seed(52); torch.cuda.manual_seed(52)
  s, nfe = fn(model, z=z.clone())
  torch.manual_seed(52); torch.cuda.manual_seed(52)
  s_host, nfe_host = fn_host(model, z=z.clone())
  assert fn.last_stats == dict(nfev=nfev, host_scalar_reads=(nfev - 2) // 6 + 3, solver='device', method='RK45')
  assert nfe == nfe_host == nfev
  assert torch.equal(s, s_host)
