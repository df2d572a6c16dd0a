"""ORACLE (test infrastructure, not product code): plain PyTorch restatement of the reference's likelihood computation
(``likelihood.py:26-113``) over the oracle SDEs (``sampling_oracle.VE / VP / SubVP``) and any ``model(x, labels)``
callable, e.g. ``ddpm_oracle.ddpm_forward`` / ``ncsnpp_oracle.ncsnpp_forward``.  The divergence is the reference's autograd
VJP, so it runs on CPU and on GPU.  Pinned against ``tests/golden/likelihood_tiny.npz``, written by the real reference
(``tools/make_golden_likelihood.py``).
"""
import numpy as np
import torch


def prior_logp(sde, z):
  """sde_lib.py:150-154 (VP), :201-204 (sub-VP), :241-244 (VE)."""
  N = np.prod(z.shape[1:])
  if sde.kind == 've':
    return -N / 2. * np.log(2 * np.pi * sde.sigma_max ** 2) - torch.sum(z ** 2, dim=(1, 2, 3)) / (2 * sde.sigma_max ** 2)
  return -N / 2. * np.log(2 * np.pi) - torch.sum(z ** 2, dim=(1, 2, 3)) / 2.


def drift(sde, model, x, t):
  """rsde.sde(x, t)[0] with probability_flow=True (sde_lib.py:93-100) over get_score_fn(continuous=True)."""
  f, g = sde.sde(x, t)
  return f - g[:, None, None, None] ** 2 * sde.score(model, x, t, True) * 0.5


def divergence(sde, model, x, t, eps):
  """get_div_fn (likelihood.py:26-37): eps . (J_drift^T eps) by autograd."""
  with torch.enable_grad():
    x = x.detach().requires_grad_(True)
    fn_eps = torch.sum(drift(sde, model, x, t) * eps)
    grad = torch.autograd.grad(fn_eps, x)[0]
  return torch.sum(grad * eps, dim=tuple(range(1, len(x.shape))))


def hutchinson_noise(data, hutchinson_type):
  """likelihood.py:84-89, the reference's own draws."""
  if hutchinson_type == 'Gaussian':
    return torch.randn_like(data)
  if hutchinson_type == 'Rademacher':
    return torch.randint_like(data, low=0, high=2).float() * 2 - 1.
  raise NotImplementedError(hutchinson_type)


def likelihood(sde, model, data, epsilon, inverse_scaler=lambda x: x, rtol=1e-5, atol=1e-5, method='RK45', eps=1e-5):
  """likelihood_fn (likelihood.py:69-111) for a given Hutchinson draw ``epsilon``.  Returns ``(bpd, z, nfe)``."""
  from scipy import integrate
  with torch.no_grad():
    shape = data.shape

    def ode_func(t, x):
      sample = torch.from_numpy(x[:-shape[0]].reshape(shape)).to(data.device).type(torch.float32)     # :92
      vec_t = torch.ones(sample.shape[0], device=sample.device) * t                                   # :93
      d = drift(sde, model, sample, vec_t).detach().cpu().numpy().reshape((-1,))                      # :94
      lg = divergence(sde, model, sample, vec_t, epsilon).detach().cpu().numpy().reshape((-1,))       # :95
      return np.concatenate([d, lg], axis=0)

    init = np.concatenate([data.detach().cpu().numpy().reshape((-1,)), np.zeros((shape[0],))], axis=0)   # :98
    solution = integrate.solve_ivp(ode_func, (eps, sde.T), init, rtol=rtol, atol=atol, method=method)
    zp = solution.y[:, -1]
    z = torch.from_numpy(zp[:-shape[0]].reshape(shape)).to(data.device).type(torch.float32)
    delta_logp = torch.from_numpy(zp[-shape[0]:].reshape((shape[0],))).to(data.device).type(torch.float32)
    bpd = -(prior_logp(sde, z) + delta_logp) / np.log(2)
    bpd = bpd / np.prod(shape[1:])
    bpd = bpd + (7. - inverse_scaler(-1.))                                                            # :108-110
    return bpd, z, solution.nfev
