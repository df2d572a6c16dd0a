"""Log-likelihood in bits/dim (``likelihood.py`` of the reference): ``get_div_fn`` and ``get_likelihood_fn`` with the same
signatures and the same ``(bpd, z, nfe)`` result.

The reference's Hutchinson-Skilling estimator is ``eps . (J_drift^T eps)``, a vector-Jacobian product through autograd
(``likelihood.py:26-35``).  For a fixed ``eps`` it equals ``eps . (J_drift eps)``, a Jacobian-vector product, and the
engine-backed networks provide that one as a forward-mode tangent pass (``EngineModel.jvp``, ``b200_ncsnpp_jvp``): no
backward graph, no stored activations.

With an engine-backed network whose configuration the tangent pass supports, an explicit Runge-Kutta ``method``
(``'RK23'``, ``'RK45'`` or ``'DOP853'``), a stock VE / VP / sub-VP SDE and CUDA data, the probability-flow ODE over the
augmented state ``[x; logp]`` is integrated device-resident (``ode.py`` + ``csrc/ode.cu``): float64 state and Runge-Kutta
stages in HBM, scipy's step-size controller on the host, one primal+tangent network evaluation per right-hand side.  The
implicit methods ``'Radau'``, ``'BDF'`` and ``'LSODA'`` (they need the Jacobian), user SDEs, CPU data and
``device_solver=False`` run the reference's loop over ``scipy.integrate.solve_ivp``; its divergence comes from autograd
for a plain ``nn.Module`` (as in the reference) and from ``model.jvp`` for an engine-backed network, whose forward has no
autograd graph.  An engine-backed network whose configuration has no tangent pass raises ``NotImplementedError``.
"""
import numpy as np
import torch
from scipy import integrate

from . import sde_lib
from .models import utils as mutils


def get_div_fn(fn):
  """Create the divergence function of `fn` using the Hutchinson-Skilling trace estimator (``likelihood.py:26-37``)."""

  def div_fn(x, t, eps):
    with torch.enable_grad():
      x.requires_grad_(True)
      fn_eps = torch.sum(fn(x, t) * eps)
      grad_fn_eps = torch.autograd.grad(fn_eps, x)[0]
    x.requires_grad_(False)
    return torch.sum(grad_fn_eps * eps, dim=tuple(range(1, len(x.shape))))

  return div_fn


def _engine_net(model):
  from . import native
  from .models._engine import EngineModel
  net = native._unwrap(model)
  if isinstance(net, EngineModel) and not net.takes_time_labels:
    raise NotImplementedError(f'likelihood: {type(net).__name__} takes noise-level indices, not the continuous-time labels '
                              'of the probability-flow ODE')
  return net if isinstance(net, EngineModel) else None


def _engine_drift_and_div(sde, net, x, t, eps):
  """Probability-flow drift (``rsde.sde(x, t)[0]``) and ``eps . (J_drift eps)`` per image for an engine-backed network:
  the score and its tangent from one ``net.jvp`` call, the SDE drift's tangent from ``torch.func.jvp`` of ``sde.sde``."""
  if isinstance(sde, (sde_lib.VPSDE, sde_lib.subVPSDE)):
    labels = t * 999                                        # models/utils.py:150 (continuous)
    out, jv = net.jvp(x, labels, eps)
    std = sde.marginal_prob(torch.zeros_like(x), t)[1]
    score, dscore = -out / std[:, None, None, None], -jv / std[:, None, None, None]
  elif isinstance(sde, sde_lib.VESDE):
    labels = sde.marginal_prob(torch.zeros_like(x), t)[1]   # models/utils.py:167
    score, dscore = net.jvp(x, labels, eps)
  else:
    raise NotImplementedError(f'SDE class {sde.__class__.__name__} not yet supported.')
  f, g = sde.sde(x, t)
  df = torch.func.jvp(lambda xx: sde.sde(xx, t)[0], (x,), (eps,))[1]
  g2 = g[:, None, None, None] ** 2
  drift = f - g2 * score * 0.5
  jdrift = df - g2 * dscore * 0.5
  # products in float64 like b200_ode_div_f64, so the host loop and the device solve see the same divergence
  return drift, torch.sum(jdrift.double() * eps.double(), dim=tuple(range(1, len(x.shape))))


def get_likelihood_fn(sde, inverse_scaler, hutchinson_type='Rademacher',
                      rtol=1e-5, atol=1e-5, method='RK45', eps=1e-5, device_solver=None):
  """Create a function to compute the unbiased log-likelihood estimate of a given data point (``likelihood.py:40-113``).

  ``device_solver``: ``None`` picks the device-resident solve when it applies, ``False`` forces the host loop, ``True``
  requires the device solve (``NotImplementedError`` otherwise).  ``likelihood_fn.last_stats`` records which solver ran
  and the method."""

  def drift_fn(model, x, t):
    """The drift function of the reverse-time SDE."""
    score_fn = mutils.get_score_fn(sde, model, train=False, continuous=True)
    # Probability flow ODE is a special case of Reverse SDE
    rsde = sde.reverse(score_fn, probability_flow=True)
    return rsde.sde(x, t)[0]

  def div_fn(model, x, t, noise):
    return get_div_fn(lambda xx, tt: drift_fn(model, xx, tt))(x, t, noise)

  def use_device_solver(net, data):
    from . import ode as _ode
    if device_solver is False:
      return False
    if device_solver and method not in _ode.METHODS:
      raise NotImplementedError(f'get_likelihood_fn(device_solver=True): method {method!r} has no device solve '
                                f'(explicit Runge-Kutta methods only: {", ".join(_ode.METHODS)})')
    ok = (net is not None and method in _ode.METHODS and data.is_cuda
          and type(sde) in (sde_lib.VESDE, sde_lib.VPSDE, sde_lib.subVPSDE))
    if device_solver and not ok:
      raise NotImplementedError('get_likelihood_fn(device_solver=True) needs an engine-backed network (NCSNpp or DDPM), '
                                "a VE/VP/sub-VP SDE and CUDA data")
    return ok

  def likelihood_fn(model, data, epsilon=None):
    """Compute an unbiased estimate to the log-likelihood in bits/dim.

    ``epsilon``: a given Hutchinson draw (same shape as ``data``) instead of the reference's own (A/B and parity tests).

    Returns:
      bpd: A PyTorch tensor of shape [batch size]. The log-likelihoods on `data` in bits/dim.
      z: A PyTorch tensor of the same shape as `data`. The latent representation of `data` under the
        probability flow ODE.
      nfe: An integer. The number of function evaluations used for running the black-box ODE solver.
    """
    with torch.no_grad():
      shape = data.shape
      if epsilon is not None:
        epsilon = epsilon.to(device=data.device, dtype=torch.float32)
      elif hutchinson_type == 'Gaussian':
        epsilon = torch.randn_like(data)
      elif hutchinson_type == 'Rademacher':
        epsilon = torch.randint_like(data, low=0, high=2).float() * 2 - 1.
      else:
        raise NotImplementedError(f"Hutchinson type {hutchinson_type} unknown.")

      net = _engine_net(model)
      if net is not None:
        net.check_jvp_supported()             # NotImplementedError before any launch: there is nothing to fall back to
      if use_device_solver(net, data):
        from . import ode as _ode
        solver = _ode.METHODS[method]
        ops = _ode.CudaOdeOps(data.to(torch.float32), _ode.engine_likelihood_fn(sde, net, epsilon.to(torch.float32)),
                              extra=shape[0], method=solver)
        nfe = solver(ops, eps, sde.T, rtol=rtol, atol=atol).solve()
        z = ops.state_f32()
        delta_logp = ops.extra_state().to(torch.float32)
        likelihood_fn.last_stats = dict(nfev=nfe, host_scalar_reads=ops.host_reads, solver='device', method=method)
      else:
        def ode_func(t, x):
          sample = mutils.from_flattened_numpy(x[:-shape[0]], shape).to(data.device).type(torch.float32)
          vec_t = torch.ones(sample.shape[0], device=sample.device) * t
          if net is not None:
            drift, div = _engine_drift_and_div(sde, net, sample, vec_t, epsilon)
            drift, logp_grad = mutils.to_flattened_numpy(drift), mutils.to_flattened_numpy(div)
          else:
            drift = mutils.to_flattened_numpy(drift_fn(model, sample, vec_t))
            logp_grad = mutils.to_flattened_numpy(div_fn(model, sample, vec_t, epsilon))
          return np.concatenate([drift, logp_grad], axis=0)

        init = np.concatenate([mutils.to_flattened_numpy(data), np.zeros((shape[0],))], axis=0)
        solution = integrate.solve_ivp(ode_func, (eps, sde.T), init, rtol=rtol, atol=atol, method=method)
        nfe = solution.nfev
        zp = solution.y[:, -1]
        z = mutils.from_flattened_numpy(zp[:-shape[0]], shape).to(data.device).type(torch.float32)
        delta_logp = mutils.from_flattened_numpy(zp[-shape[0]:], (shape[0],)).to(data.device).type(torch.float32)
        likelihood_fn.last_stats = dict(nfev=nfe, solver='scipy', method=method)
      prior_logp = sde.prior_logp(z)
      bpd = -(prior_logp + delta_logp) / np.log(2)
      N = np.prod(shape[1:])
      bpd = bpd / N
      # A hack to convert log-likelihoods to bits/dim
      offset = 7. - inverse_scaler(-1.)
      bpd = bpd + offset
      return bpd, z, nfe

  return likelihood_fn
