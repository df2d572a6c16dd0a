"""Inpainting and colorization with PC samplers — mirror of ``controllable_generation.py:8-198``.

Same factories, signatures and results: ``get_pc_inpainter(...) -> pc_inpainter(model, data, mask)`` and
``get_pc_colorizer(...) -> pc_colorizer(model, gray_scale_img)``.  Both are the PC loop of ``sampling.py`` with one extra
step after every corrector / predictor update: the known part of the image (the masked pixels, or the luminance channel
of an orthonormal colour transform) is replaced by a fresh draw from the forward marginal of the data at time ``t``.
RNG consumption follows the reference draw for draw (prior sample, then per update: the update's own noise, then
``randn_like`` for the data marginal).

Where ``native.match_pc_plan`` accepts the sampler (an engine-backed model on CUDA, a stock SDE, stock predictor and
corrector, ``continuous=True``) the ``sde.N`` iterations run on the native PC loop: one CUDA graph per iteration, the
blend in one kernel (``pc_constrain_kernel``) with its noise generated in-kernel from the same Philox stream.  Any other
combination (user modules or update classes, ``continuous=False``) runs the host loop below over this package's
``shared_*_update_fn``.  ``pc_inpainter.last_stats`` / ``pc_colorizer.last_stats`` record which loop ran.
"""
import functools

import torch

from .sampling import shared_corrector_update_fn, shared_predictor_update_fn

# Orthonormal colour transform of ``controllable_generation.py:109-111``: channel 0 of ``decouple(x)`` is the grey level.
_M = ((5.7735014e-01, -8.1649649e-01, 4.7008697e-08),
      (5.7735026e-01, 4.0824834e-01, 7.0710671e-01),
      (5.7735026e-01, 4.0824822e-01, -7.0710683e-01))


def _update_fns(sde, predictor, corrector, snr, n_steps, probability_flow, continuous):
  pred = functools.partial(shared_predictor_update_fn, sde=sde, predictor=predictor, probability_flow=probability_flow,
                           continuous=continuous)
  corr = functools.partial(shared_corrector_update_fn, sde=sde, corrector=corrector, continuous=continuous, snr=snr,
                           n_steps=n_steps)
  return corr, pred


def _native_plan(constraint, model, x, sde, predictor, corrector, snr, n_steps, probability_flow, continuous, eps):
  """The native constrained plan for the initial state ``x``, or ``None`` when the host loop has to run.

  ``torch.randn_like(x)`` fills a dense tensor in memory order, and every update keeps the initial state's layout
  (the state is always the first operand).  The colorizer's state is the output of an einsum, which is channels-last
  for batches > 1, so its draws land in NHWC order; the plan is told which order the reference's draws take."""
  if not x.is_cuda or x.dtype != torch.float32:
    return None
  if x.is_contiguous():
    channels_last = False
  elif x.is_contiguous(memory_format=torch.channels_last):
    channels_last = True
  else:
    return None
  from . import native  # late import: the native library is only needed for engine models
  return native.match_pc_plan(sde=sde, model=model, predictor=predictor, corrector=corrector, shape=x.shape, snr=snr,
                              n_steps=n_steps, probability_flow=probability_flow, continuous=continuous, eps=eps,
                              device=x.device, constraint=constraint, channels_last=channels_last)


def _constrained_pc_loop(sde, model, x, known, mask, update_fns, to_latent, from_latent, eps):
  """``sde.N`` iterations of (corrector, predictor), each followed by the data-consistency step
  (``controllable_generation.py:43-52`` / ``:137-146``): in the latent space given by ``to_latent``, the coordinates
  selected by ``mask`` are overwritten with a noisy copy of ``known`` at the current noise level.  As in the reference,
  ``x_mean`` is rebuilt from the *blended* ``x`` (not from the update's own mean)."""
  timesteps = torch.linspace(sde.T, eps, sde.N)
  x_mean = x
  for i in range(sde.N):
    t = timesteps[i]
    for update_fn in update_fns:
      vec_t = torch.ones(x.shape[0], device=x.device) * t
      x, _ = update_fn(x, vec_t, model=model)
      known_mean, std = sde.marginal_prob(known, vec_t)
      known_noisy = known_mean + torch.randn_like(x) * std[:, None, None, None]
      x = from_latent(to_latent(x) * (1. - mask) + known_noisy * mask)
      x_mean = from_latent(to_latent(x) * (1. - mask) + known_mean * mask)
  return x, x_mean


def get_pc_inpainter(sde, predictor, corrector, inverse_scaler, snr, n_steps=1, probability_flow=False, continuous=False,
                     denoise=True, eps=1e-5):
  """``controllable_generation.py:8-80``.  ``mask`` is 1 on known pixels, 0 where the image is to be generated."""
  update_fns = _update_fns(sde, predictor, corrector, snr, n_steps, probability_flow, continuous)
  ident = lambda v: v

  def pc_inpainter(model, data, mask):
    with torch.no_grad():
      x = data * mask + sde.prior_sampling(data.shape).to(data.device) * (1. - mask)
      plan = None
      if x.shape == data.shape:   # a mask that would broadcast the data to a larger shape stays on the host loop
        plan = _native_plan('inpaint', model, x, sde, predictor, corrector, snr, n_steps, probability_flow, continuous,
                            eps)
      if plan is not None:
        x, x_mean = plan.run(x, data, mask)
        pc_inpainter.last_stats = dict(loop='native', launches_per_step=plan.launches_per_step())
      else:
        x, x_mean = _constrained_pc_loop(sde, model, x, data, mask, update_fns, ident, ident, eps)
        pc_inpainter.last_stats = dict(loop='host')
      return inverse_scaler(x_mean if denoise else x)

  return pc_inpainter


def get_pc_colorizer(sde, predictor, corrector, inverse_scaler, snr, n_steps=1, probability_flow=False, continuous=False,
                     denoise=True, eps=1e-5):
  """``controllable_generation.py:83-198``.  ``gray_scale_img`` has identical R, G, B channels."""
  update_fns = _update_fns(sde, predictor, corrector, snr, n_steps, probability_flow, continuous)
  M = torch.tensor(_M)
  invM = torch.inverse(M)
  decouple = lambda v: torch.einsum('bihw,ij->bjhw', v, M.to(v.device))
  couple = lambda v: torch.einsum('bihw,ij->bjhw', v, invM.to(v.device))

  def pc_colorizer(model, gray_scale_img):
    with torch.no_grad():
      g = gray_scale_img
      mask = torch.cat([torch.ones_like(g[:, :1, ...]), torch.zeros_like(g[:, 1:, ...])], dim=1)
      x = couple(decouple(g) * mask + decouple(sde.prior_sampling(g.shape).to(g.device) * (1. - mask)))
      plan = _native_plan('colorize', model, x, sde, predictor, corrector, snr, n_steps, probability_flow, continuous, eps)
      if plan is not None:
        x, x_mean = plan.run(x, decouple(g), mask)
        pc_colorizer.last_stats = dict(loop='native', launches_per_step=plan.launches_per_step())
      else:
        x, x_mean = _constrained_pc_loop(sde, model, x, decouple(g), mask, update_fns, decouple, couple, eps)
        pc_colorizer.last_stats = dict(loop='host')
      return inverse_scaler(x_mean if denoise else x)

  return pc_colorizer
