"""CPU tests for the losses oracle and the op-gradient oracle against goldens written by the REAL reference
(tools/make_golden_f4.py), and the host logic of score_sde_pytorch_b200.losses (no device work)."""
import numpy as np
import pytest
import torch

from helpers import golden, golden_config, seeded_model
from oracle import losses_oracle as LO
from oracle import ncsnpp_oracle as NO
from oracle import sampling_oracle as SO
from tools_f4_cases import FIR_CASES, StandIn

SDES = {'ve': lambda: SO.VE(0.01, 50, 1000), 'vp': lambda: SO.VP(0.1, 20, 1000), 'subvp': lambda: SO.SubVP(0.1, 20, 1000)}


def _net(cfg):
  sd = seeded_model(cfg).state_dict()
  return lambda x, labels: NO.ncsnpp_forward(sd, cfg, x, labels)


@pytest.mark.parametrize('mname,sname', [('tiny', 've'), ('tiny_vp', 'vp'), ('tiny_vp', 'subvp'), ('tiny_ddpmpp', 'vp')])
def test_oracle_sde_losses_match_the_reference(mname, sname):
  g = golden('f4_losses.npz')
  cfg = golden_config(mname)
  net, sde = _net(cfg), SDES[sname]()
  batch = torch.from_numpy(g[f'{mname}_batch'])
  t, z = torch.from_numpy(g[f'{mname}_{sname}_t']), torch.from_numpy(g[f'{mname}_{sname}_z'])
  with torch.no_grad():
    for rm in (False, True):
      for lw in (False, True):
        loss, _ = LO.sde_loss(sde, lambda x, tt: sde.score(net, x, tt), batch, t, z, reduce_mean=rm, likelihood_weighting=lw)
        ref = float(g[f'{mname}_{sname}_loss_rm{int(rm)}_lw{int(lw)}'])
        assert abs(loss.item() - ref) <= 2e-6 * abs(ref), (mname, sname, rm, lw, loss.item(), ref)


def test_oracle_ddpm_loss_matches_the_reference():
  g = golden('f4_losses.npz')
  cfg = golden_config('tiny_ddpmpp')
  net, sde = _net(cfg), SO.VP(0.1, 20, 1000)
  batch = torch.from_numpy(g['tiny_ddpmpp_batch'])
  labels, z = torch.from_numpy(g['tiny_ddpmpp_ddpm_labels']), torch.from_numpy(g['tiny_ddpmpp_ddpm_z'])
  sa = torch.sqrt(torch.cumprod(sde.alphas, dim=0))
  with torch.no_grad():
    for rm in (False, True):
      loss, _ = LO.ddpm_loss(sa, sde.sqrt_1m_alphas_cumprod, net, batch, labels, z, reduce_mean=rm)
      ref = float(g[f'tiny_ddpmpp_ddpm_loss_rm{int(rm)}'])
      assert abs(loss.item() - ref) <= 2e-6 * abs(ref)


def test_oracle_smld_loss_matches_the_reference():
  """get_smld_loss_fn (losses.py:105-126) on a deterministic stand-in model: the loss arithmetic (descending sigma table,
  perturbation, target -noise / sigma^2, reduction, sigma^2 weighting) is what is pinned."""
  g = golden('f4_losses.npz')
  sde = SO.VE(0.01, 50, 1000)
  batch = torch.from_numpy(g['smld_batch'])
  labels, z = torch.from_numpy(g['smld_labels']), torch.from_numpy(g['smld_z'])
  with torch.no_grad():
    for rm in (False, True):
      loss, _ = LO.smld_loss(torch.flip(sde.discrete_sigmas, dims=(0,)), StandIn(), batch, labels, z, reduce_mean=rm)
      ref = float(g[f'smld_loss_rm{int(rm)}'])
      assert abs(loss.item() - ref) <= 2e-6 * abs(ref), (rm, loss.item(), ref)


@pytest.mark.parametrize('case', FIR_CASES, ids=lambda c: c[0])
def test_oracle_upfirdn2d_gradients_match_the_reference(case):
  name = case[0]
  g = golden('f4_op_grads.npz')
  up, down, p0, p1 = (int(v) for v in g[f'fir_{name}_cfg'])
  t = lambda k: torch.from_numpy(g[f'fir_{name}_{k}'])
  y, gi, ggo = LO.upfirdn2d_grads(t('x'), t('k'), up, down, (p0, p1), t('go'), t('v'))
  for got, key in ((y, 'y'), (gi, 'gi'), (ggo, 'ggo')):
    assert got.shape == t(key).shape
    assert torch.allclose(got, t(key), rtol=1e-6, atol=1e-6), (name, key)


def test_oracle_fused_leaky_relu_gradients_match_the_reference():
  g = golden('f4_op_grads.npz')
  t = lambda k: torch.from_numpy(g[f'lrelu_{k}'])
  y, gi, gb, ggo = LO.fused_leaky_relu_grads(t('x'), t('b'), t('go'), t('vi'), t('vb'))
  for got, key in ((y, 'y'), (gi, 'gi'), (gb, 'gb'), (ggo, 'ggo')):
    assert torch.allclose(got, t(key), rtol=1e-6, atol=1e-6), key


def test_losses_module_host_logic():
  """Training needs the network backward: every train=True constructor raises; CPU batches are rejected (no CPU path);
  the optimizer plumbing follows losses.py:25-52 (Adam fields, linear warm-up, gradient clipping)."""
  from score_sde_pytorch_b200 import losses, sde_lib
  sde = sde_lib.VESDE(0.01, 50, 1000)
  for make in (lambda: losses.get_sde_loss_fn(sde, train=True), lambda: losses.get_smld_loss_fn(sde, train=True),
               lambda: losses.get_ddpm_loss_fn(sde_lib.VPSDE(), train=True), lambda: losses.get_step_fn(sde, train=True)):
    with pytest.raises(NotImplementedError, match='backward'):
      make()
  with pytest.raises(AssertionError):
    losses.get_smld_loss_fn(sde_lib.VPSDE(), train=False)
  with pytest.raises(AssertionError):
    losses.get_ddpm_loss_fn(sde, train=False)
  with pytest.raises(ValueError, match='not recommended'):
    losses.get_step_fn(sde_lib.subVPSDE(), train=False, continuous=False)
  with pytest.raises(RuntimeError, match='CUDA'):
    losses.get_sde_loss_fn(sde, train=False)(None, torch.zeros(2, 3, 8, 8))
  cfg = golden_config('tiny')
  cfg.optim.lr, cfg.optim.warmup, cfg.optim.grad_clip = 2e-4, 5000, 1.0
  w = torch.nn.Parameter(torch.ones(10))
  opt = losses.get_optimizer(cfg, [w])
  d = opt.defaults
  assert (d['lr'], d['betas'], d['eps'], d['weight_decay']) == (cfg.optim.lr, (cfg.optim.beta1, 0.999), cfg.optim.eps, cfg.optim.weight_decay)
  cfg.optim.optimizer = 'SGD'
  with pytest.raises(NotImplementedError):
    losses.get_optimizer(cfg, [w])
  cfg.optim.optimizer = 'Adam'
  w.grad = torch.full((10,), 3.0)
  losses.optimization_manager(cfg)(opt, [w], step=1000)
  assert abs(opt.param_groups[0]['lr'] - 2e-4 * 0.2) < 1e-12                 # warm-up: lr * step / warmup
  assert abs(w.grad.norm().item() - 1.0) < 1e-5                              # clipped to max_norm = grad_clip
  assert (w.detach() < 1).all()                                              # and a step was taken
