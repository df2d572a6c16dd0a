"""CPU tests of the device ODE solver's host logic for scipy's three explicit Runge-Kutta methods (RK23, RK45, DOP853):
the restated step-size controller (score_sde_pytorch_b200/ode.py) driven by a numpy `ops` that does scipy's own array
arithmetic must reproduce scipy.integrate.solve_ivp(method=m) bit for bit - same nfev, same accepted times, same final
state.  Also: the tableaux are scipy's, the DOP853 reduction is exported, and the implicit methods keep the scipy path."""
import math

import numpy as np
import pytest
import torch
from scipy import integrate

from score_sde_pytorch_b200 import ode as O


class ScipyArithmeticOps:
  """``ops`` with the exact numpy expressions of scipy's rk_step, _estimate_error_norm and select_initial_step; the sums
  of squares are ``x.dot(x)``, which is what ``np.linalg.norm`` squares."""

  def __init__(self, y0, fun, method):
    self.method = method
    self.y = np.asarray(y0, dtype=np.float64).copy()
    self.n = self.y.size
    self.y_new = np.empty_like(self.y)
    self.K = np.empty((method.n_stages + 1, self.n))
    self.fun = fun
    self.solver = None
    self.accepted_t = []

  def rhs(self, t, coefs, h, slot, keep_y):
    s = len(coefs)
    ys = self.y + np.dot(self.K[:s].T, np.asarray(coefs)) * h if s else self.y
    if keep_y:
      self.y_new = ys.copy()
    self.K[slot] = self.fun(t, ys)

  def _scale(self, rtol, atol):
    return atol + np.maximum(np.abs(self.y), np.abs(self.y_new)) * rtol

  def error_sumsq(self, h, rtol, atol):
    x = np.dot(self.K.T, np.asarray(self.method.E)) * h / self._scale(rtol, atol)
    return float(x.dot(x))

  def error_sumsq2(self, rtol, atol):
    scale = self._scale(rtol, atol)
    e5 = np.dot(self.K.T, np.asarray(self.method.E5)) / scale
    e3 = np.dot(self.K.T, np.asarray(self.method.E3)) / scale
    return float(e5.dot(e5)), float(e3.dot(e3))

  def scaled_sumsq(self, slot, minus, rtol, atol):
    v = self.y if slot < 0 else self.K[slot]
    if minus is not None:
      v = v - self.K[minus]
    x = v / (atol + np.abs(self.y) * rtol)
    return float(x.dot(x))

  def accept(self):
    self.y, self.y_new = self.y_new, self.y
    self.K[0] = self.K[self.method.n_stages]
    self.accepted_t.append(self.solver.t)


def smooth_problem(n=257):
  rng = np.random.default_rng(3)
  w = rng.normal(size=n).astype(np.float32)
  y0 = rng.normal(size=n).astype(np.float32)        # the reference hands solve_ivp a float32 array (to_flattened_numpy)

  def fun(t, y):                                    # float32 right-hand side widened to float64, like the reference's ode_func
    x = y.astype(np.float32)
    return (-(1.5 + np.float32(t)) * x + np.sin(3 * x + w) * np.float32(4.0)).astype(np.float32).astype(np.float64)

  return y0, fun


def kicked_problem(n=300):
  """Ten stiff components (rate 300) that hold every method at its stability limit, and a pulse in time at t = 1.2:
  each method has to reject steps (8 to 27 of them on these cases)."""
  rng = np.random.default_rng(8)
  y0 = rng.normal(size=n)
  a = rng.uniform(0.5, 2.0, size=n)
  a[:10] = 300.0

  def fun(t, y):
    return -a * y + 40.0 * np.exp(-((t - 1.2) / 0.05) ** 2) * np.cos(y)

  return y0, fun


CASES = [('smooth', (1.0, 1e-3), 1e-5), ('smooth', (1.0, 1e-3), 1e-3), ('smooth', (0.0, 2.5), 1e-5),
         ('smooth', (0.0, 2.5), 1e-3), ('kicked', (0.0, 2.0), 1e-6), ('kicked', (0.0, 2.0), 1e-4)]


@pytest.mark.parametrize('name', ['RK23', 'RK45', 'DOP853'])
@pytest.mark.parametrize('problem,span,tol', CASES)
def test_controller_reproduces_scipy_solve_ivp_bit_for_bit(name, problem, span, tol):
  y0, fun = smooth_problem() if problem == 'smooth' else kicked_problem()
  # the controller divides by math.sqrt(n), scipy by n ** 0.5 (libm pow): the same double for these sizes
  assert math.sqrt(y0.size) == y0.size ** 0.5
  sol = integrate.solve_ivp(fun, span, y0, rtol=tol, atol=tol, method=name)
  assert sol.status == 0
  method = O.METHODS[name]
  ops = ScipyArithmeticOps(y0, fun, method)
  solver = method(ops, span[0], span[1], rtol=tol, atol=tol)
  ops.solver = solver
  nfev = solver.solve()
  assert nfev == sol.nfev
  assert ops.accepted_t == sol.t[1:].tolist()
  assert np.array_equal(ops.y, sol.y[:, -1])
  if problem == 'kicked':
    assert solver.n_rejected > 0


def test_tableaux_are_scipys():
  for name, cls in (('RK23', integrate.RK23), ('RK45', integrate.RK45), ('DOP853', integrate.DOP853)):
    m = O.METHODS[name]
    assert m.name == name
    assert (m.order, m.error_estimator_order, m.n_stages) == (cls.order, cls.error_estimator_order, cls.n_stages)
    assert np.array_equal(np.asarray(m.C), cls.C)
    assert np.array_equal(np.asarray(m.B), cls.B)
    assert len(m.A) == m.n_stages
    full = np.zeros(cls.A.shape)                        # (6, 5) for RK45, square otherwise
    for s, row in enumerate(m.A):
      assert len(row) == s
      full[s, :s] = row
    assert np.array_equal(full, cls.A)                  # scipy's A is strictly lower triangular
    if name == 'DOP853':
      assert np.array_equal(np.asarray(m.E5), cls.E5) and np.array_equal(np.asarray(m.E3), cls.E3)
      assert len(m.E5) == m.n_stages + 1 <= 16           # b200_ode_error_sumsq2_f64 takes at most 16 weights
    else:
      assert np.array_equal(np.asarray(m.E), cls.E) and len(m.E) == m.n_stages + 1


def test_rk45_tableau_is_unchanged():
  """DormandPrince45 and the module-level names keep the Dormand-Prince 5(4) doubles they had as literals."""
  assert O.METHODS['RK45'] is O.DormandPrince45
  assert O.C == (0.0, 1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0)
  assert O.A == ((), (1 / 5,), (3 / 40, 9 / 40), (44 / 45, -56 / 15, 32 / 9),
                 (19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729),
                 (9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656))
  assert O.B == (35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84)
  assert O.E == (-71 / 57600, 0.0, 71 / 16695, -71 / 1920, 17253 / 339200, -22 / 525, 1 / 40)
  assert (O.ORDER, O.ERROR_ESTIMATOR_ORDER, O.N_STAGES) == (5, 4, 6)


def test_dop853_reduction_is_exported():
  from score_sde_pytorch_b200 import _lib
  lib = _lib.load()
  assert hasattr(lib, 'b200_ode_error_sumsq2_f64')
  assert lib.b200_ode_workspace_doubles() >= 2 * 1024 + 8


class Linear(torch.nn.Module):
  """A plain module, ``model(x, labels)``: x -> -x."""

  def forward(self, x, labels):
    return -x


def test_sampler_routes_implicit_methods_to_scipy():
  from score_sde_pytorch_b200 import sampling, sde_lib
  sde = sde_lib.VPSDE(0.1, 20., 1000)
  shape = (1, 1, 2, 2)
  z = torch.linspace(-1, 1, 4).reshape(shape)
  fn = sampling.get_ode_sampler(sde, shape, lambda v: v, method='Radau', rtol=1e-3, atol=1e-3, device='cpu')
  x, nfe = fn(Linear(), z=z.clone())
  assert fn.last_stats == dict(nfev=nfe, solver='scipy', method='Radau')
  assert torch.isfinite(x).all()
  for method in ('Radau', 'BDF', 'LSODA'):
    fn = sampling.get_ode_sampler(sde, shape, lambda v: v, method=method, device='cpu', device_solver=True)
    with pytest.raises(NotImplementedError, match=method):
      fn(Linear(), z=z.clone())


def test_likelihood_routes_implicit_methods_to_scipy():
  from score_sde_pytorch_b200 import likelihood, sde_lib
  sde = sde_lib.VPSDE(0.1, 20., 1000)
  data = torch.linspace(-1, 1, 4).reshape(1, 1, 2, 2)
  fn = likelihood.get_likelihood_fn(sde, lambda v: v, method='Radau', rtol=1e-3, atol=1e-3)
  torch.manual_seed(0)
  bpd, z, nfe = fn(Linear(), data)
  assert fn.last_stats == dict(nfev=nfe, solver='scipy', method='Radau')
  assert torch.isfinite(bpd).all()
  for method in ('Radau', 'BDF', 'LSODA'):
    fn = likelihood.get_likelihood_fn(sde, lambda v: v, method=method, device_solver=True)
    with pytest.raises(NotImplementedError, match=method):
      fn(Linear(), data)
