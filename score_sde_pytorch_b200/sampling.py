"""Predictor–corrector and ODE samplers.

Mirror of the reference's ``sampling.py`` surface — registries (``:30-77``),
``get_sampling_fn`` (``:80-123``), ``Predictor``/``Corrector`` ABCs
(``:126-173``), the shipped predictors/correctors (``:176-331``),
``shared_{predictor,corrector}_update_fn`` (``:333-352``), ``get_pc_sampler``
(``:355-411``) and ``get_ode_sampler`` (``:414-485``) — with one structural
change: ``pc_sampler(model)`` first asks :mod:`score_sde_pytorch_b200.native`
whether ``(sde, predictor, corrector, model)`` is a combination the sm_90a
engine implements (an engine-backed NCSN++ on a CUDA device with the
reverse-diffusion / Euler–Maruyama / none predictor and the Langevin / none
corrector).  If so the whole loop — both network evaluations, the in-kernel
Philox noise, the Langevin norms and both state updates of every step — runs
as a replayed CUDA graph with no Python in the loop.  Anything else (user
models, user predictor/corrector classes, CPU tensors) runs the generic host
loop below, which keeps the reference's extension points working
(``README.md:119-122``).
"""
import abc
import functools

import numpy as np
import torch

from . import sde_lib
from .models import utils as mutils
from .models.utils import from_flattened_numpy, to_flattened_numpy, get_score_fn

_CORRECTORS = {}
_PREDICTORS = {}


def _make_register(table):
  def register(cls=None, *, name=None):
    def _register(c):
      key = c.__name__ if name is None else name
      if key in table:
        raise ValueError(f'Already registered model with name: {key}')
      table[key] = c
      return c
    return _register if cls is None else _register(cls)
  return register


register_predictor = _make_register(_PREDICTORS)
register_predictor.__doc__ = "Decorator registering a Predictor class (``sampling.py:34-50``)."
register_corrector = _make_register(_CORRECTORS)
register_corrector.__doc__ = "Decorator registering a Corrector class (``sampling.py:53-69``)."


def get_predictor(name):
  return _PREDICTORS[name]


def get_corrector(name):
  return _CORRECTORS[name]


def get_sampling_fn(config, sde, shape, inverse_scaler, eps):
  """Build ``sampling_fn(model) -> (samples, nfe)`` from ``config.sampling``
  (``sampling.py:80-123``).  Unknown sampler names raise ``ValueError``."""
  method = config.sampling.method.lower()
  if method == 'ode':
    return get_ode_sampler(sde=sde, shape=shape, inverse_scaler=inverse_scaler,
                           denoise=config.sampling.noise_removal, eps=eps, device=config.device)
  if method == 'pc':
    return get_pc_sampler(sde=sde, shape=shape,
                          predictor=get_predictor(config.sampling.predictor.lower()),
                          corrector=get_corrector(config.sampling.corrector.lower()),
                          inverse_scaler=inverse_scaler, snr=config.sampling.snr,
                          n_steps=config.sampling.n_steps_each,
                          probability_flow=config.sampling.probability_flow,
                          continuous=config.training.continuous,
                          denoise=config.sampling.noise_removal, eps=eps, device=config.device)
  if method == 'dpm_solver':
    smp = config.sampling
    return get_dpm_solver_sampler(sde=sde, shape=shape, inverse_scaler=inverse_scaler,
                                  steps=getattr(smp, 'dpm_steps', 20), order=getattr(smp, 'dpm_order', 3),
                                  algorithm=getattr(smp, 'dpm_algorithm', 'dpmsolver++'),
                                  skip_type=getattr(smp, 'dpm_skip_type', 'logSNR'),
                                  denoise=smp.noise_removal, eps=eps, device=config.device)
  raise ValueError(f"Sampler name {config.sampling.method} unknown.")


class Predictor(abc.ABC):
  """Abstract predictor: one step of the reverse-time SDE/ODE (``sampling.py:126-148``)."""

  def __init__(self, sde, score_fn, probability_flow=False):
    super().__init__()
    self.sde = sde
    self.rsde = sde.reverse(score_fn, probability_flow)
    self.score_fn = score_fn

  @abc.abstractmethod
  def update_fn(self, x, t):
    """Return ``(x_next, x_next_mean)``."""


class Corrector(abc.ABC):
  """Abstract corrector: score-based MCMC at fixed ``t`` (``sampling.py:151-173``)."""

  def __init__(self, sde, score_fn, snr, n_steps):
    super().__init__()
    self.sde = sde
    self.score_fn = score_fn
    self.snr = snr
    self.n_steps = n_steps

  @abc.abstractmethod
  def update_fn(self, x, t):
    """Return ``(x_next, x_next_mean)``."""


def _col(v):
  return v[:, None, None, None]


@register_predictor(name='euler_maruyama')
class EulerMaruyamaPredictor(Predictor):
  """``x' = x + drift·dt + g·sqrt(-dt)·z`` with ``dt = -1/N`` (``sampling.py:176-187``)."""

  def update_fn(self, x, t):
    dt = -1. / self.rsde.N
    z = torch.randn_like(x)
    drift, diffusion = self.rsde.sde(x, t)
    x_mean = x + drift * dt
    return x_mean + _col(diffusion) * np.sqrt(-dt) * z, x_mean


@register_predictor(name='reverse_diffusion')
class ReverseDiffusionPredictor(Predictor):
  """``x' = x − f_rev + G·z`` from ``rsde.discretize`` (``sampling.py:190-200``)."""

  def update_fn(self, x, t):
    f, G = self.rsde.discretize(x, t)
    z = torch.randn_like(x)
    x_mean = x - f
    return x_mean + _col(G) * z, x_mean


@register_predictor(name='ancestral_sampling')
class AncestralSamplingPredictor(Predictor):
  """Ancestral sampling for VE / VP (``sampling.py:203-239``)."""

  def __init__(self, sde, score_fn, probability_flow=False):
    super().__init__(sde, score_fn, probability_flow)
    if not isinstance(sde, (sde_lib.VPSDE, sde_lib.VESDE)):
      raise NotImplementedError(f"SDE class {sde.__class__.__name__} not yet supported.")
    assert not probability_flow, "Probability flow not supported by ancestral sampling"

  def vesde_update_fn(self, x, t):
    sde = self.sde
    idx = (t * (sde.N - 1) / sde.T).long()
    table = sde.discrete_sigmas.to(t.device)
    sigma = table[idx]
    adjacent = torch.where(idx == 0, torch.zeros_like(t), table[idx - 1])
    score = self.score_fn(x, t)
    x_mean = x + score * _col(sigma ** 2 - adjacent ** 2)
    std = torch.sqrt((adjacent ** 2 * (sigma ** 2 - adjacent ** 2)) / (sigma ** 2))
    return x_mean + _col(std) * torch.randn_like(x), x_mean

  def vpsde_update_fn(self, x, t):
    sde = self.sde
    idx = (t * (sde.N - 1) / sde.T).long()
    beta = sde.discrete_betas.to(t.device)[idx]
    score = self.score_fn(x, t)
    x_mean = (x + _col(beta) * score) / _col(torch.sqrt(1. - beta))
    return x_mean + _col(torch.sqrt(beta)) * torch.randn_like(x), x_mean

  def update_fn(self, x, t):
    if isinstance(self.sde, sde_lib.VESDE):
      return self.vesde_update_fn(x, t)
    return self.vpsde_update_fn(x, t)


@register_predictor(name='none')
class NonePredictor(Predictor):
  """Identity predictor (corrector-only sampling)."""

  def __init__(self, sde, score_fn, probability_flow=False):
    pass

  def update_fn(self, x, t):
    return x, x


def _langevin_alpha(sde, t):
  if isinstance(sde, (sde_lib.VPSDE, sde_lib.subVPSDE)):
    idx = (t * (sde.N - 1) / sde.T).long()
    return sde.alphas.to(t.device)[idx]
  return torch.ones_like(t)


def _check_corrector_sde(sde):
  if not isinstance(sde, (sde_lib.VPSDE, sde_lib.VESDE, sde_lib.subVPSDE)):
    raise NotImplementedError(f"SDE class {sde.__class__.__name__} not yet supported.")


@register_corrector(name='langevin')
class LangevinCorrector(Corrector):
  """Langevin MCMC whose step size is set from the **batch-mean** gradient and
  noise norms (``sampling.py:253-282``; the means at ``:276-277`` couple all
  images of a batch through one scalar)."""

  def __init__(self, sde, score_fn, snr, n_steps):
    super().__init__(sde, score_fn, snr, n_steps)
    _check_corrector_sde(sde)

  def update_fn(self, x, t):
    alpha = _langevin_alpha(self.sde, t)
    x_mean = x
    for _ in range(self.n_steps):
      grad = self.score_fn(x, t)
      noise = torch.randn_like(x)
      grad_norm = torch.norm(grad.reshape(grad.shape[0], -1), dim=-1).mean()
      noise_norm = torch.norm(noise.reshape(noise.shape[0], -1), dim=-1).mean()
      step_size = (self.snr * noise_norm / grad_norm) ** 2 * 2 * alpha
      x_mean = x + _col(step_size) * grad
      x = x_mean + _col(torch.sqrt(step_size * 2)) * noise
    return x, x_mean


@register_corrector(name='ald')
class AnnealedLangevinDynamics(Corrector):
  """NCSN-style annealed Langevin dynamics (``sampling.py:285-319``)."""

  def __init__(self, sde, score_fn, snr, n_steps):
    super().__init__(sde, score_fn, snr, n_steps)
    _check_corrector_sde(sde)

  def update_fn(self, x, t):
    alpha = _langevin_alpha(self.sde, t)
    std = self.sde.marginal_prob(x, t)[1]
    x_mean = x
    for _ in range(self.n_steps):
      grad = self.score_fn(x, t)
      noise = torch.randn_like(x)
      step_size = (self.snr * std) ** 2 * 2 * alpha
      x_mean = x + _col(step_size) * grad
      x = x_mean + noise * _col(torch.sqrt(step_size * 2))
    return x, x_mean


@register_corrector(name='none')
class NoneCorrector(Corrector):
  """Identity corrector (predictor-only sampling)."""

  def __init__(self, sde, score_fn, snr, n_steps):
    pass

  def update_fn(self, x, t):
    return x, x


def shared_predictor_update_fn(x, t, sde, model, predictor, probability_flow, continuous):
  """Configure a predictor on ``model`` and apply one update (``sampling.py:333-341``)."""
  score_fn = mutils.get_score_fn(sde, model, train=False, continuous=continuous)
  cls = NonePredictor if predictor is None else predictor
  return cls(sde, score_fn, probability_flow).update_fn(x, t)


def shared_corrector_update_fn(x, t, sde, model, corrector, continuous, snr, n_steps):
  """Configure a corrector on ``model`` and apply one update (``sampling.py:344-352``)."""
  score_fn = mutils.get_score_fn(sde, model, train=False, continuous=continuous)
  cls = NoneCorrector if corrector is None else corrector
  return cls(sde, score_fn, snr, n_steps).update_fn(x, t)


def get_pc_sampler(sde, shape, predictor, corrector, inverse_scaler, snr,
                   n_steps=1, probability_flow=False, continuous=False,
                   denoise=True, eps=1e-3, device='cuda'):
  """Create ``pc_sampler(model) -> (samples, nfe)`` (``sampling.py:355-411``).

  ``predictor`` / ``corrector`` are classes (or ``None``).  ``nfe`` is reported as
  ``sde.N * (n_steps + 1)`` exactly as the reference does (``:409``), including
  when a None predictor/corrector makes the true count smaller.
  """
  predictor_update_fn = functools.partial(shared_predictor_update_fn, sde=sde, predictor=predictor,
                                          probability_flow=probability_flow, continuous=continuous)
  corrector_update_fn = functools.partial(shared_corrector_update_fn, sde=sde, corrector=corrector,
                                          continuous=continuous, snr=snr, n_steps=n_steps)

  def pc_sampler(model):
    from . import native  # late import: the native library is only needed for engine models
    plan = native.match_pc_plan(sde=sde, model=model, predictor=predictor, corrector=corrector,
                                shape=shape, snr=snr, n_steps=n_steps,
                                probability_flow=probability_flow, continuous=continuous,
                                eps=eps, device=device)
    with torch.no_grad():
      x = sde.prior_sampling(shape).to(device)
      if plan is not None:
        x, x_mean = plan.run(x)
      else:
        timesteps = torch.linspace(sde.T, eps, sde.N, device=device)
        x_mean = x
        for i in range(sde.N):
          vec_t = torch.ones(shape[0], device=timesteps.device) * timesteps[i]
          x, x_mean = corrector_update_fn(x, vec_t, model=model)
          x, x_mean = predictor_update_fn(x, vec_t, model=model)
      return inverse_scaler(x_mean if denoise else x), sde.N * (n_steps + 1)

  return pc_sampler


def _denoise_update(sde, model, x, eps):
  """One reverse-diffusion predictor step at ``t = eps`` without noise: the ``noise_removal`` step of the ODE samplers
  (``sampling.py:433-441``)."""
  score_fn = get_score_fn(sde, model, train=False, continuous=True)
  vec_eps = torch.ones(x.shape[0], device=x.device) * eps
  return ReverseDiffusionPredictor(sde, score_fn, probability_flow=False).update_fn(x, vec_eps)[1]


def get_ode_sampler(sde, shape, inverse_scaler, denoise=False, rtol=1e-5, atol=1e-5,
                    method='RK45', eps=1e-3, device='cuda', device_solver=None):
  """Probability-flow ODE sampler (``sampling.py:414-485``): same signature, same ``(samples, nfe)`` result.

  With an engine-backed network (NCSN++ or DDPM) on a CUDA device, an explicit Runge-Kutta ``method`` (``'RK23'``,
  ``'RK45'`` or ``'DOP853'``) and a stock VE / VP / sub-VP SDE the solve is device-resident (``ode.py`` + ``csrc/ode.cu``):
  float64 state and Runge-Kutta stages in HBM, scipy's step-size controller on the host, one transfer of the error sums
  per attempted step.  Anything else - user models or SDEs, the implicit methods ``'Radau'``, ``'BDF'`` and ``'LSODA'``
  (they need the Jacobian) - runs the reference's host loop over ``scipy.integrate.solve_ivp`` (each right-hand side then
  crosses PCIe twice, as in the reference).  ``device_solver=False`` forces the host loop (A/B and parity tests);
  ``device_solver=True`` requires the device solve (``NotImplementedError`` otherwise).  ``ode_sampler.last_stats``
  records which solver ran and the method."""

  def denoise_update_fn(model, x):
    return _denoise_update(sde, model, x, eps)

  def drift_fn(model, x, t):
    score_fn = get_score_fn(sde, model, train=False, continuous=True)
    return sde.reverse(score_fn, probability_flow=True).sde(x, t)[0]

  def use_device_solver(model, x):
    from . import native, ode as _ode
    if device_solver is False:
      return False
    if method not in _ode.METHODS:
      if device_solver:
        raise NotImplementedError(f'get_ode_sampler(device_solver=True): method {method!r} has no device solve '
                                  f'(explicit Runge-Kutta methods only: {", ".join(_ode.METHODS)})')
      return False
    if not x.is_cuda:
      return False
    from .models._engine import EngineModel
    net = native._unwrap(model)
    ok = isinstance(net, EngineModel) and type(sde) in (sde_lib.VESDE, sde_lib.VPSDE, sde_lib.subVPSDE)
    if ok and not net.takes_time_labels:
      raise NotImplementedError(f'get_ode_sampler: {type(net).__name__} takes noise-level indices, not the continuous-time '
                                'labels of the probability-flow ODE')
    if device_solver and not ok:
      raise NotImplementedError('get_ode_sampler(device_solver=True) needs an engine-backed network (NCSNpp or DDPM) and a '
                                'VE/VP/sub-VP SDE')
    return ok

  def ode_sampler(model, z=None):
    with torch.no_grad():
      x = sde.prior_sampling(shape).to(device) if z is None else z
      if use_device_solver(model, x):
        from . import native, ode as _ode
        net = native._unwrap(model)
        solver = _ode.METHODS[method]
        ops = _ode.CudaOdeOps(x.reshape(shape).to(torch.float32), _ode.engine_drift_fn(sde, net, shape[0], x.device),
                              method=solver)
        nfe = solver(ops, sde.T, eps, rtol=rtol, atol=atol).solve()
        x = ops.state_f32()
        ode_sampler.last_stats = dict(nfev=nfe, host_scalar_reads=ops.host_reads, solver='device', method=method)
      else:
        from scipy import integrate

        def ode_func(t, flat):
          xt = from_flattened_numpy(flat, shape).to(device).type(torch.float32)
          vec_t = torch.ones(shape[0], device=xt.device) * t
          return to_flattened_numpy(drift_fn(model, xt, vec_t))

        sol = integrate.solve_ivp(ode_func, (sde.T, eps), to_flattened_numpy(x),
                                  rtol=rtol, atol=atol, method=method)
        x = torch.tensor(sol.y[:, -1]).reshape(shape).to(device).type(torch.float32)
        nfe = sol.nfev
        ode_sampler.last_stats = dict(nfev=nfe, solver='scipy', method=method)
      if denoise:
        x = denoise_update_fn(model, x)
      return inverse_scaler(x), nfe

  return ode_sampler


def get_dpm_solver_sampler(sde, shape, inverse_scaler, steps=20, order=3, algorithm='dpmsolver++', skip_type='logSNR',
                           denoise=False, eps=1e-3, device='cuda'):
  """Multistep DPM-Solver (``algorithm='dpmsolver'``, noise prediction; Lu et al., arXiv:2206.00927) or DPM-Solver++
  (``'dpmsolver++'``, data prediction; arXiv:2211.01095) sampler of the probability-flow ODE from ``sde.T`` to ``eps``:
  ``steps`` network evaluations at ``order`` 1 (DDIM), 2 or 3 on a grid uniform in log-SNR (``skip_type='logSNR'``), in
  ``t`` (``'time_uniform'``) or in ``sqrt(t)`` (``'time_quadratic'``); tables from :func:`native.build_multistep_tables`.
  The network is evaluated as ``get_ode_sampler`` evaluates it (``get_score_fn(..., continuous=True)``) and ``denoise``
  adds the same final ``noise_removal`` step (one more evaluation).

  Returns ``sampler(model, z=None) -> (samples, nfe)``.  With an engine network that takes time labels on a CUDA device
  the loop is native (one CUDA-graph replay per step: the forward and one fused update kernel); any other ``nn.Module``
  runs an eager host loop over the same tables in the dtype of the state.  ``sampler.last_stats`` records ``loop``
  (``'native'`` / ``'host'``), ``steps``, ``order`` and ``nfe``.  Raises ``ValueError`` for an ``order`` outside 1-3,
  ``steps < 1`` or an unknown ``algorithm`` / ``skip_type``, and ``NotImplementedError`` for SDEs other than VESDE,
  VPSDE and subVPSDE and for networks that take noise-level indices (NCSNv2)."""
  from . import native
  tab = native.build_multistep_tables(sde, steps, order, algorithm, skip_type, eps)

  def host_loop(model, x):
    score_fn = get_score_fn(sde, model, train=False, continuous=True)
    prev = []                                   # M_{i-1}, M_{i-2}
    for i in range(steps):
      vec_t = torch.full((x.shape[0],), float(tab['t'][i]), dtype=x.dtype, device=x.device)
      m = float(tab['mq'][i]) * x + float(tab['ms'][i]) * score_fn(x, vec_t)
      xn = float(tab['pa'][i]) * x + float(tab['pb'][i]) * m
      for c, mp in zip((tab['pm1'][i], tab['pm2'][i]), prev):
        if c != 0:
          xn = xn + float(c) * mp
      prev = [m] + prev[:1]
      x = xn
    return x

  def dpm_solver_sampler(model, z=None):
    from .models._engine import EngineModel
    net = native._unwrap(model)
    if isinstance(net, EngineModel) and not net.takes_time_labels:
      raise NotImplementedError(f'get_dpm_solver_sampler: {type(net).__name__} takes noise-level indices, not the '
                                'continuous-time labels of the probability-flow ODE')
    with torch.no_grad():
      x = sde.prior_sampling(shape).to(device) if z is None else z
      plan = native.match_multistep_plan(sde, model, shape, steps, order, algorithm, skip_type, eps, x.device) \
          if x.is_cuda else None
      if plan is not None:
        x, _ = plan.run(x.to(torch.float32))
      else:
        x = host_loop(model, x)
      nfe = steps + int(bool(denoise))
      if denoise:
        x = _denoise_update(sde, model, x, eps)
      dpm_solver_sampler.last_stats = dict(loop='host' if plan is None else 'native', steps=steps, order=order, nfe=nfe)
      return inverse_scaler(x), nfe

  return dpm_solver_sampler
