"""Device-resident probability-flow ODE solver (successor of the host-side scipy loops of ``sampling.py:414-485`` and
``likelihood.py:84-113``).

``scipy.integrate.solve_ivp(method=m)`` keeps the state in a float64 numpy array and calls the right-hand side with it:
in the reference every function evaluation moves the whole batch host -> device -> host.  Here the float64 state, the
Runge-Kutta stage derivatives and every stage / error sum live in HBM (``csrc/ode.cu`` behind ``b200_ode_*``); this
module is scipy's step-size CONTROLLER restated on Python floats (IEEE doubles, like numpy's): ``select_initial_step``
(``scipy/integrate/_ivp/common.py``), ``RungeKutta._step_impl``, ``_estimate_error_norm`` and ``rk_step``
(``_ivp/rk.py``), and ``solve_ivp``'s outer loop without events / dense output.  It covers scipy's three explicit
Runge-Kutta pairs, with scipy's own coefficient arrays:

  ``RK23``    Bogacki-Shampine 3(2): 3 stages + FSAL, error estimator order 2
  ``RK45``    Dormand-Prince 5(4): 6 stages + FSAL, error estimator order 4 (:class:`DormandPrince45`)
  ``DOP853``  Dormand-Prince 8(5,3): 12 stages + FSAL, error estimator order 7, scipy's combined 5th/3rd-order error norm

One transfer per attempted step crosses PCIe (the sum of squares behind the error norm; for DOP853 the two sums of its
two estimators); the accepted/rejected decision is taken on the host exactly as scipy takes it, so the trajectory of step
sizes - and ``nfev`` - follow scipy's for the same right-hand side.  ``Radau``, ``BDF`` and ``LSODA`` are implicit
methods that need the Jacobian of the right-hand side; they have no device solve.

:class:`RungeKutta` is arithmetic-agnostic: it drives an ``ops`` object (``CudaOdeOps`` below; the CPU tests plug a
numpy one in to compare the controller with scipy itself).
"""
import ctypes
import math

import torch
from scipy import integrate as _scipy

from . import _lib


def _tableau(cls):
  """(C, A, B) of a scipy ``RungeKutta`` class as Python floats; row s of A holds the s coefficients ``rk_step`` uses."""
  return (tuple(float(c) for c in cls.C), tuple(tuple(float(a) for a in cls.A[s, :s]) for s in range(cls.n_stages)),
          tuple(float(b) for b in cls.B))


SAFETY, MIN_FACTOR, MAX_FACTOR = 0.9, 0.2, 10.0     # _ivp/rk.py module constants


class RungeKutta:
  """``ops`` provides (all state stays wherever ``ops`` keeps it; K[j] is stage-derivative slot j of n_stages + 1):
      ops.n                                  number of state elements
      ops.rhs(t, coefs, h, slot, keep_y)     K[slot] = f(t, y + h * sum_j coefs[j] K[j]); keep_y: also store that state as y_new
      ops.error_sumsq(h, rtol, atol)         sum(((h * sum_j E[j] K[j]) / (atol + max(|y|, |y_new|) * rtol))**2)
      ops.error_sumsq2(rtol, atol)           DOP853 only: the same sum without h for E5 and for E3, as a pair
      ops.scaled_sumsq(slot, minus, rtol, atol)   sum(((K[slot] - K[minus]) / (atol + |y| * rtol))**2), slot=-1: y itself
      ops.accept()                           y <- y_new, K[0] <- K[n_stages]

  The norm divides by ``math.sqrt(n)``; scipy's ``x.size ** 0.5`` goes through libm's ``pow``, which for about 0.1 % of
  sizes rounds differently in the last bit."""
  name = None
  C = A = B = E = None
  order = error_estimator_order = n_stages = None

  def __init__(self, ops, t0, t_bound, rtol=1e-5, atol=1e-5, max_step=math.inf):
    self.ops, self.t, self.t_bound = ops, float(t0), float(t_bound)
    self.rtol, self.atol, self.max_step = float(rtol), float(atol), max_step
    self.direction = (1.0 if t_bound > t0 else -1.0) if t_bound != t0 else 1.0
    self.error_exponent = -1 / (self.error_estimator_order + 1)
    self.nfev = 0
    self.n_accepted = self.n_rejected = 0
    self._rhs(self.t, (), 0.0, 0, False)                      # self.f = self.fun(self.t, self.y)
    self.h_abs = self._select_initial_step()

  def _rhs(self, t, coefs, h, slot, keep_y):
    self.nfev += 1
    self.ops.rhs(t, coefs, h, slot, keep_y)

  def _norm(self, sumsq):
    return math.sqrt(sumsq) / math.sqrt(self.ops.n)           # np.linalg.norm(x) / x.size ** 0.5

  def _error_norm(self, h):
    """RungeKutta._estimate_error_norm(K, h, scale)."""
    return self._norm(self.ops.error_sumsq(h, self.rtol, self.atol))

  def _select_initial_step(self):
    """scipy/integrate/_ivp/common.py:select_initial_step (order = error_estimator_order)."""
    interval_length = abs(self.t_bound - self.t)
    if interval_length == 0.0:
      return 0.0
    d0 = self._norm(self.ops.scaled_sumsq(-1, None, self.rtol, self.atol))
    d1 = self._norm(self.ops.scaled_sumsq(0, None, self.rtol, self.atol))
    h0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    h0 = min(h0, interval_length)
    self._rhs(self.t + h0 * self.direction, (1.0,), h0 * self.direction, 1, False)      # f1 = fun(t0 + h0*dir, y0 + h0*dir*f0)
    d2 = self._norm(self.ops.scaled_sumsq(1, 0, self.rtol, self.atol)) / h0
    if d1 <= 1e-15 and d2 <= 1e-15:
      h1 = max(1e-6, h0 * 1e-3)
    else:
      h1 = (0.01 / max(d1, d2)) ** (1 / (self.error_estimator_order + 1))
    return min(100 * h0, h1, interval_length, self.max_step)

  def _step(self):
    """RungeKutta._step_impl + rk_step.  Returns False if the step size underflowed."""
    t = self.t
    min_step = 10 * abs(math.nextafter(t, self.direction * math.inf) - t)
    if self.h_abs > self.max_step:
      h_abs = self.max_step
    elif self.h_abs < min_step:
      h_abs = min_step
    else:
      h_abs = self.h_abs
    step_accepted = step_rejected = False
    while not step_accepted:
      if h_abs < min_step:
        return False
      h = h_abs * self.direction
      t_new = t + h
      if self.direction * (t_new - self.t_bound) > 0:
        t_new = self.t_bound
      h = t_new - t
      h_abs = abs(h)
      for s in range(1, self.n_stages):                        # rk_step: K[s] = fun(t + c*h, y + (K[:s].T @ a[:s]) * h)
        self._rhs(t + self.C[s] * h, self.A[s], h, s, False)
      self._rhs(t + h, self.B, h, self.n_stages, True)         # y_new = y + h * K[:-1].T @ B; K[-1] = fun(t + h, y_new)
      error_norm = self._error_norm(h)
      if error_norm < 1:
        factor = MAX_FACTOR if error_norm == 0 else min(MAX_FACTOR, SAFETY * error_norm ** self.error_exponent)
        if step_rejected:
          factor = min(1, factor)
        h_abs *= factor
        step_accepted = True
        self.n_accepted += 1
      else:
        h_abs *= max(MIN_FACTOR, SAFETY * error_norm ** self.error_exponent)
        step_rejected = True
        self.n_rejected += 1
    self.t = t_new
    self.ops.accept()
    self.h_abs = h_abs
    return True

  def solve(self):
    """solve_ivp's loop (no events, no dense output): step until t_bound.  Returns nfev."""
    while self.direction * (self.t - self.t_bound) < 0:
      if not self._step():
        raise RuntimeError(f'{self.name}: required step size is less than spacing between numbers')   # solve_ivp status -1
    return self.nfev


class RK23(RungeKutta):
  """scipy.integrate.RK23: Bogacki-Shampine 3(2)."""
  name = 'RK23'
  order, error_estimator_order, n_stages = _scipy.RK23.order, _scipy.RK23.error_estimator_order, _scipy.RK23.n_stages
  C, A, B = _tableau(_scipy.RK23)
  E = tuple(float(e) for e in _scipy.RK23.E)


class DormandPrince45(RungeKutta):
  """scipy.integrate.RK45: Dormand-Prince 5(4)."""
  name = 'RK45'
  order, error_estimator_order, n_stages = _scipy.RK45.order, _scipy.RK45.error_estimator_order, _scipy.RK45.n_stages
  C, A, B = _tableau(_scipy.RK45)
  E = tuple(float(e) for e in _scipy.RK45.E)


class DOP853(RungeKutta):
  """scipy.integrate.DOP853: Dormand-Prince 8(5,3), whose error norm combines a 5th- and a 3rd-order estimator."""
  name = 'DOP853'
  order, error_estimator_order, n_stages = _scipy.DOP853.order, _scipy.DOP853.error_estimator_order, _scipy.DOP853.n_stages
  C, A, B = _tableau(_scipy.DOP853)
  E5 = tuple(float(e) for e in _scipy.DOP853.E5)
  E3 = tuple(float(e) for e in _scipy.DOP853.E3)

  def _error_norm(self, h):
    """DOP853._estimate_error_norm: |h| ||err5||^2 / sqrt((||err5||^2 + 0.01 ||err3||^2) n), err = K.E / scale."""
    s5, s3 = self.ops.error_sumsq2(self.rtol, self.atol)
    err5_norm_2, err3_norm_2 = math.sqrt(s5) ** 2, math.sqrt(s3) ** 2       # np.linalg.norm(err) ** 2
    if err5_norm_2 == 0 and err3_norm_2 == 0:
      return 0.0
    denom = err5_norm_2 + 0.01 * err3_norm_2
    return abs(h) * err5_norm_2 / math.sqrt(denom * self.ops.n)


# the explicit methods of solve_ivp, by the name it takes
METHODS = {'RK23': RK23, 'RK45': DormandPrince45, 'DOP853': DOP853}

# Dormand-Prince 5(4) tableau under its earlier module-level names
C, A, B, E = DormandPrince45.C, DormandPrince45.A, DormandPrince45.B, DormandPrince45.E
ORDER, ERROR_ESTIMATOR_ORDER, N_STAGES = DormandPrince45.order, DormandPrince45.error_estimator_order, DormandPrince45.n_stages


class CudaOdeOps:
  """The float64 state ``y`` / ``y_new``, the stage derivatives ``K[n_stages + 1][n]`` and the float32 network input on
  the device.  ``drift(t, x32, k_out)`` (given by the sampler) evaluates the network on ``x32`` and writes the float64
  drift.  ``method`` is the controller class (a value of :data:`METHODS`) whose tableau the ops evaluate.

  ``extra`` > 0 appends that many zero-initialised float64 entries to the state (the likelihood ODE's ``logp`` slots,
  ``likelihood.py:98``): ``x32`` is then the image part of the float32 stage state and ``k_out`` the whole stage row.

  Memory: n_stages + 3 float64 copies of the state plus one float32 copy.  For a CIFAR-10 likelihood state at batch 1024
  (n = 1024 * 3072 + 1024 = 3,146,752 doubles, 25.2 MB each) that is 176 MB of stages for RK45 (7 rows), 101 MB for RK23
  (4 rows) and 327 MB for DOP853 (13 rows); with y, y_new and x32 DOP853 holds 390 MB."""

  def __init__(self, x0, drift, extra=0, method=DormandPrince45):
    self.method = method
    self.device = x0.device
    self.shape = tuple(x0.shape)
    self.n_img = x0.numel()
    y = x0.detach().to(torch.float64).reshape(-1)
    if extra:
      y = torch.cat([y, torch.zeros(extra, dtype=torch.float64, device=self.device)])
    self.n = y.numel()
    self.y = y.contiguous()
    self.y_new = torch.empty_like(self.y)
    self.K = torch.empty(method.n_stages + 1, self.n, dtype=torch.float64, device=self.device)
    self.x32_flat = torch.empty(self.n, dtype=torch.float32, device=self.device)
    self.x32 = self.x32_flat[:self.n_img].view(self.shape)
    self.ws = torch.zeros(int(_lib.load().b200_ode_workspace_doubles()), dtype=torch.float64, device=self.device)
    self.drift = drift
    self.host_reads = 0

  def _coefs(self, coefs):
    arr = (ctypes.c_double * 16)()
    for j, c in enumerate(coefs):
      arr[j] = c
    return arr

  def rhs(self, t, coefs, h, slot, keep_y):
    st = _lib.stream_ptr(self.device)
    _lib.call('b200_ode_stage_f64', _lib.ptr(self.y), _lib.ptr(self.K), self.n, self._coefs(coefs), len(coefs), float(h),
              _lib.ptr(self.y_new) if keep_y else None, _lib.ptr(self.x32_flat), st)
    self.drift(t, self.x32, self.K[slot])

  def _read(self):
    self.host_reads += 1
    return float(self.ws[0].item())          # the one device -> host scalar

  def error_sumsq(self, h, rtol, atol):
    e = self.method.E
    _lib.call('b200_ode_error_sumsq_f64', _lib.ptr(self.y), _lib.ptr(self.y_new), _lib.ptr(self.K), self.n, self._coefs(e),
              len(e), float(h), float(rtol), float(atol), _lib.ptr(self.ws), _lib.stream_ptr(self.device))
    return self._read()

  def error_sumsq2(self, rtol, atol):
    e5, e3 = self.method.E5, self.method.E3
    _lib.call('b200_ode_error_sumsq2_f64', _lib.ptr(self.y), _lib.ptr(self.y_new), _lib.ptr(self.K), self.n,
              self._coefs(e5), self._coefs(e3), len(e5), float(rtol), float(atol), _lib.ptr(self.ws),
              _lib.stream_ptr(self.device))
    self.host_reads += 1
    s5, s3 = self.ws[:2].tolist()            # one device -> host copy of the two sums
    return s5, s3

  def scaled_sumsq(self, slot, minus, rtol, atol):
    v = self.y if slot < 0 else self.K[slot]
    v2 = None if minus is None else self.K[minus]
    _lib.call('b200_ode_scaled_sumsq_f64', _lib.ptr(v), _lib.ptr(v2), _lib.ptr(self.y), self.n, float(rtol), float(atol),
              _lib.ptr(self.ws), _lib.stream_ptr(self.device))
    return self._read()

  def accept(self):
    self.y, self.y_new = self.y_new, self.y
    self.K[0].copy_(self.K[self.method.n_stages])      # FSAL: self.f = f_new

  def state_f32(self):
    return self.y[:self.n_img].to(torch.float32).reshape(self.shape)

  def extra_state(self):
    """The appended float64 entries of the state (``extra`` > 0)."""
    return self.y[self.n_img:].clone()


def engine_drift_fn(sde, model, batch, device):
  """Right-hand side of the probability-flow ODE for the engine-backed network and the stock VE / VP / sub-VP SDEs:
  ``rsde.sde(x, t)[0]`` with ``probability_flow=True`` (``sde_lib.py:93-100``) over ``get_score_fn(..., continuous=True)``
  (``models/utils.py:129-178``).  The per-evaluation scalars - network label, drift coefficient, g(t)^2, marginal std -
  come from the SDE's own torch ops on a one-element device tensor and stay on the device."""
  from . import sde_lib
  vp_like = isinstance(sde, (sde_lib.VPSDE, sde_lib.subVPSDE))
  one = torch.ones(1, 1, 1, 1, device=device)
  zero = torch.zeros(1, 1, 1, 1, device=device)
  scal = torch.zeros(3, dtype=torch.float32, device=device)

  def drift(t, x32, k_out):
    vec_t = torch.ones(1, device=device) * t                       # `torch.ones(shape[0]) * t`: float32
    f1, g = sde.sde(one, vec_t)                                    # drift of x = 1 (the drift is linear in x), diffusion
    std = sde.marginal_prob(zero, vec_t)[1]
    if vp_like:
      labels = vec_t * 999                                         # models/utils.py:150
      scal[2:3] = std
    else:
      labels = std                                                 # VE: labels = sigma(t) (:167), score = model output
      scal[2] = 0.0
    scal[0:1] = f1.reshape(1)
    scal[1:2] = g ** 2
    out = model(x32, labels.to(torch.float32).expand(batch).contiguous(), labels_uniform=True)
    _lib.call('b200_ode_drift_f64', _lib.ptr(x32), _lib.ptr(out), x32.numel(), _lib.ptr(scal), _lib.ptr(k_out),
              _lib.stream_ptr(device))

  return drift


def engine_likelihood_fn(sde, model, epsilon):
  """Right-hand side of the likelihood ODE (``likelihood.py:91-96``) over the augmented state ``[x; logp]`` for the
  engine-backed network: one ``b200_ncsnpp_jvp`` evaluation gives the network output and ``J_net eps``; the drift goes to
  ``k_out[:n]`` (``b200_ode_drift_f64``, as the ODE sampler) and the per-image divergence ``eps . (J_drift eps)`` to the
  logp slots ``k_out[n:]`` (``b200_ode_div_f64``).  Scalars as in :func:`engine_drift_fn`."""
  from . import sde_lib
  vp_like = isinstance(sde, (sde_lib.VPSDE, sde_lib.subVPSDE))
  device = epsilon.device
  batch = epsilon.shape[0]
  n = epsilon.numel()
  eps = epsilon.contiguous()
  one = torch.ones(1, 1, 1, 1, device=device)
  zero = torch.zeros(1, 1, 1, 1, device=device)
  scal = torch.zeros(3, dtype=torch.float32, device=device)

  def rhs(t, x32, k_out):
    vec_t = torch.ones(1, device=device) * t
    f1, g = sde.sde(one, vec_t)
    std = sde.marginal_prob(zero, vec_t)[1]
    if vp_like:
      labels = vec_t * 999
      scal[2:3] = std
    else:
      labels = std
      scal[2] = 0.0
    scal[0:1] = f1.reshape(1)
    scal[1:2] = g ** 2
    out, jv = model.jvp(x32, labels.to(torch.float32).expand(batch).contiguous(), eps, labels_uniform=True)
    st = _lib.stream_ptr(device)
    _lib.call('b200_ode_drift_f64', _lib.ptr(x32), _lib.ptr(out), n, _lib.ptr(scal), _lib.ptr(k_out), st)
    _lib.call('b200_ode_div_f64', _lib.ptr(eps), _lib.ptr(jv), batch, n // batch, _lib.ptr(scal), _lib.ptr(k_out[n:]), st)

  return rhs
