"""Score-matching losses and the evaluation step — mirror of the reference's ``losses.py``.

Surface: ``get_optimizer`` (``losses.py:25-34``), ``optimization_manager`` (``:37-52``), ``get_sde_loss_fn``
(``:55-102``), ``get_smld_loss_fn`` (``:105-126``), ``get_ddpm_loss_fn`` (``:129-148``), ``get_step_fn`` (``:151-210``).

What runs where.  The EVALUATION loss (``train=False``: run_lib.py's eval step and the loss part of ``evaluate``) is a
device path: the batch is perturbed by ``b200_dsm_perturb_f32``, the score network is the engine's forward, the squared
residual is reduced per image by ``b200_dsm_loss_f32`` (csrc/losses.cu); the per-image scalars (mean coefficient, std,
sigma, g^2) come from the SDE's own torch ops on ``[B]`` tensors, and ``t`` / ``z`` are drawn from torch's generator in the
reference's order (``t`` first, then ``z``), so a CUDA seed gives the draws the reference would make on that device.
The TRAINING step needs the network's backward pass and dropout, which the engine does not have: ``train=True`` raises
``NotImplementedError``.  The optimizer plumbing is host logic and is mirrored so
that configs and checkpoints carry over.

``loss_fn(model, batch, t=None, z=None)``: the two extra arguments replace the internal draws (tests pin the loss to
the reference's value on the reference's own CPU draws this way).
"""
import numpy as np
import torch
import torch.optim as optim

from . import _lib, sde_lib
from .models import utils as mutils
from .sde_lib import VESDE, VPSDE


def get_optimizer(config, params):
  """Adam with the config's learning rate, ``(beta1, 0.999)``, eps and weight decay (``losses.py:25-34``)."""
  if config.optim.optimizer == 'Adam':
    return optim.Adam(params, lr=config.optim.lr, betas=(config.optim.beta1, 0.999), eps=config.optim.eps,
                      weight_decay=config.optim.weight_decay)
  raise NotImplementedError(f'Optimizer {config.optim.optimizer} not supported yet!')


def optimization_manager(config):
  """``optimize_fn(optimizer, params, step)``: linear warm-up of the learning rate, gradient-norm clipping (disabled when
  negative), optimizer step (``losses.py:37-52``)."""

  def optimize_fn(optimizer, params, step, lr=config.optim.lr, warmup=config.optim.warmup, grad_clip=config.optim.grad_clip):
    if warmup > 0:
      for g in optimizer.param_groups:
        g['lr'] = lr * np.minimum(step / warmup, 1.0)
    if grad_clip >= 0:
      torch.nn.utils.clip_grad_norm_(params, max_norm=grad_clip)
    optimizer.step()

  return optimize_fn


def _no_training(what):
  raise NotImplementedError(f'{what}: train=True needs the backward pass and dropout of the score network, which the sm_90a '
                            'engine does not implement (evaluation losses and sampling only)')


def _perturb(batch, z, mean_coef, noise_coef):
  """``mean_coef[:, None, None, None] * batch + noise_coef[:, None, None, None] * z`` on the device library."""
  x = batch.detach().to(torch.float32).contiguous()
  zz = z.detach().to(torch.float32).contiguous()
  out = torch.empty_like(x)
  a = None if mean_coef is None else mean_coef.detach().to(torch.float32).contiguous()
  s = noise_coef.detach().to(torch.float32).contiguous()
  with torch.cuda.device(x.device):
    _lib.call('b200_dsm_perturb_f32', _lib.ptr(x), _lib.ptr(zz), _lib.ptr(a), _lib.ptr(s), _lib.ptr(out), x.shape[0],
              x[0].numel(), _lib.stream_ptr(x.device))
  return out


def _reduce(score, z, w, w2, mode, reduce_mean):
  """Per-image ``reduce(residual ** 2)`` (``b200_dsm_loss_f32``): ``[B]`` float32."""
  sc = score.detach().to(torch.float32).contiguous()
  zz = z.detach().to(torch.float32).contiguous()
  B, n = sc.shape[0], sc[0].numel()
  lib = _lib.load()
  ws = torch.empty(int(lib.b200_dsm_workspace_doubles(B, n)), dtype=torch.float64, device=sc.device)
  out = torch.empty(B, dtype=torch.float32, device=sc.device)
  f = lambda t: None if t is None else t.detach().to(torch.float32).contiguous()
  w, w2 = f(w), f(w2)
  with torch.cuda.device(sc.device):
    _lib.call('b200_dsm_loss_f32', _lib.ptr(sc), _lib.ptr(zz), _lib.ptr(w), _lib.ptr(w2), _lib.ptr(out), B, n, mode,
              1 if reduce_mean else 0, _lib.ptr(ws), _lib.stream_ptr(sc.device))
  return out


def _require_cuda(batch):
  if not batch.is_cuda:
    raise RuntimeError('losses (score_sde_pytorch_b200): batch must be a CUDA tensor (no CPU path)')


def get_sde_loss_fn(sde, train, reduce_mean=True, continuous=True, likelihood_weighting=True, eps=1e-5):
  """Denoising score matching for a continuous-time SDE (``losses.py:55-102``): ``t ~ U(eps, T)``, ``z ~ N(0, I)``,
  ``x_t = mean(x, t) + std(t) z``; the per-image loss is ``reduce((score * std + z)^2)``, or with likelihood weighting
  ``reduce((score + z / std)^2) * g(t)^2``; ``reduce`` = mean, or half the sum; the result is the batch mean."""
  if train:
    _no_training('get_sde_loss_fn')

  def loss_fn(model, batch, t=None, z=None):
    _require_cuda(batch)
    score_fn = mutils.get_score_fn(sde, model, train=False, continuous=continuous)
    B = batch.shape[0]
    with torch.no_grad():
      if t is None:
        t = torch.rand(B, device=batch.device) * (sde.T - eps) + eps
      if z is None:
        z = torch.randn_like(batch)
      one = torch.ones(B, 1, 1, 1, device=batch.device)
      mean_coef, std = sde.marginal_prob(one, t)           # the marginal mean is linear in x for every SDE of sde_lib
      perturbed = _perturb(batch, z, mean_coef.reshape(B), std)
      score = score_fn(perturbed, t)
      if not likelihood_weighting:
        losses = _reduce(score, z, std, None, 0, reduce_mean)
      else:
        g2 = sde.sde(torch.zeros(B, 1, 1, 1, device=batch.device), t)[1] ** 2
        losses = _reduce(score, z, std, None, 1, reduce_mean) * g2
      return torch.mean(losses)

  return loss_fn


def get_smld_loss_fn(vesde, train, reduce_mean=False):
  """Legacy SMLD objective on the discrete noise levels of a VE SDE (``losses.py:105-126``)."""
  assert isinstance(vesde, VESDE), "SMLD training only works for VESDEs."
  if train:
    _no_training('get_smld_loss_fn')
  smld_sigma_array = torch.flip(vesde.discrete_sigmas, dims=(0,))   # earlier SMLD models count sigmas downwards

  def loss_fn(model, batch, labels=None, z=None):
    _require_cuda(batch)
    model_fn = mutils.get_model_fn(model, train=False)
    with torch.no_grad():
      if labels is None:
        labels = torch.randint(0, vesde.N, (batch.shape[0],), device=batch.device)
      sigmas = smld_sigma_array.to(batch.device)[labels]
      if z is None:
        z = torch.randn_like(batch)
      perturbed = _perturb(batch, z, None, sigmas)         # noise + batch, noise = z * sigma
      score = model_fn(perturbed, labels)
      losses = _reduce(score, z, sigmas, sigmas ** 2, 2, reduce_mean) * sigmas ** 2
      return torch.mean(losses)

  return loss_fn


def get_ddpm_loss_fn(vpsde, train, reduce_mean=True):
  """Legacy DDPM objective on the discrete steps of a VP SDE (``losses.py:129-148``)."""
  assert isinstance(vpsde, VPSDE), "DDPM training only works for VPSDEs."
  if train:
    _no_training('get_ddpm_loss_fn')

  def loss_fn(model, batch, labels=None, z=None):
    _require_cuda(batch)
    model_fn = mutils.get_model_fn(model, train=False)
    with torch.no_grad():
      if labels is None:
        labels = torch.randint(0, vpsde.N, (batch.shape[0],), device=batch.device)
      a = vpsde.sqrt_alphas_cumprod.to(batch.device)[labels]
      s = vpsde.sqrt_1m_alphas_cumprod.to(batch.device)[labels]
      if z is None:
        z = torch.randn_like(batch)
      perturbed = _perturb(batch, z, a, s)
      score = model_fn(perturbed, labels)
      return torch.mean(_reduce(score, z, None, None, 3, reduce_mean))

  return loss_fn


def get_step_fn(sde, train, optimize_fn=None, reduce_mean=False, continuous=True, likelihood_weighting=False):
  """One evaluation step (``losses.py:151-210`` with ``train=False``): the loss of the EMA weights on a batch - the
  model's parameters are stored, overwritten with the averages (which repacks the engine's weights), evaluated and put
  back.  ``state`` is the reference's dict (``model``, ``ema``, ``step``, ``optimizer``)."""
  if train:
    _no_training('get_step_fn')
  if continuous:
    loss_fn = get_sde_loss_fn(sde, train, reduce_mean=reduce_mean, continuous=True, likelihood_weighting=likelihood_weighting)
  else:
    assert not likelihood_weighting, "Likelihood weighting is not supported for original SMLD/DDPM training."
    if isinstance(sde, VESDE):
      loss_fn = get_smld_loss_fn(sde, train, reduce_mean=reduce_mean)
    elif isinstance(sde, VPSDE):
      loss_fn = get_ddpm_loss_fn(sde, train, reduce_mean=reduce_mean)
    else:
      raise ValueError(f"Discrete training for {sde.__class__.__name__} is not recommended.")

  def step_fn(state, batch):
    model = state['model']
    with torch.no_grad():
      ema = state['ema']
      ema.store(model.parameters())
      ema.copy_to(model.parameters())
      loss = loss_fn(model, batch)
      ema.restore(model.parameters())
    return loss

  return step_fn
