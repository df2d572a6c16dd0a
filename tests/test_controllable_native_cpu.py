"""CPU: the host side of controllable generation on the native PC loop - the blend's per-step tables, the C ABI
additions, and the host-loop choice for models the native loop does not cover."""
import ctypes

import numpy as np
import pytest
import torch

from score_sde_pytorch_b200 import _lib, native, sde_lib


@pytest.mark.parametrize('kind', ['ve', 'vp', 'subvp'])
def test_constraint_tables_equal_marginal_prob_as_the_reference_evaluates_it(kind):
  """cm[i] * known and cs[i] are sde.marginal_prob(known, vec_t) at t_i = linspace(T, eps, N)[i], with vec_t a batch of
  t_i as in controllable_generation.py:42-45."""
  sde = {'ve': lambda: sde_lib.VESDE(0.01, 50, 17), 'vp': lambda: sde_lib.VPSDE(0.1, 20., 17),
         'subvp': lambda: sde_lib.subVPSDE(0.1, 20., 17)}[kind]()
  eps = 1e-3
  tab = native.build_constraint_tables(sde, eps)
  assert tab['cm'].dtype == np.float32 and tab['cs'].dtype == np.float32 and tab['cm'].shape == (17,)
  torch.manual_seed(0)
  known = torch.randn(4, 3, 5, 5)
  timesteps = torch.linspace(sde.T, eps, sde.N)
  for i in range(sde.N):
    vec_t = torch.ones(known.shape[0]) * timesteps[i]
    mean, std = sde.marginal_prob(known, vec_t)
    assert torch.equal(mean, torch.from_numpy(tab['cm'])[i] * known), i
    assert torch.equal(std, torch.full_like(std, float(tab['cs'][i]))), i
  if kind == 've':
    assert (tab['cm'] == 1).all()


def test_bind_constraint_symbol_is_exported():
  lib = _lib.load()
  assert hasattr(lib, 'b200_pc_bind_constraint')
  assert 'b200_pc_bind_constraint' in _lib.SIGNATURES


def test_unconstrained_pc_config_defaults_leave_constraint_off():
  cfg = _lib.PcConfig()
  assert cfg.constraint == 0 and not cfg.cm and not cfg.cs
  assert list(cfg.color_m) == [0.0] * 9 and list(cfg.color_minv) == [0.0] * 9
  # the new fields trail the existing ones, so the old layout is a prefix of the new one
  assert _lib.PcConfig.constraint.offset > _lib.PcConfig.cc.offset
  assert _lib.PcConfig.color_minv.offset + 9 * ctypes.sizeof(ctypes.c_float) <= ctypes.sizeof(_lib.PcConfig)


def test_plain_module_runs_the_host_loop():
  from score_sde_pytorch_b200 import controllable_generation as CG, sampling

  class Zero(torch.nn.Module):
    def forward(self, x, labels):
      return torch.zeros_like(x)

  sde = sde_lib.VESDE(0.01, 50, 3)
  kw = dict(snr=0.16, n_steps=1, probability_flow=False, continuous=True, denoise=True, eps=1e-5)
  inp = CG.get_pc_inpainter(sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, lambda v: v, **kw)
  col = CG.get_pc_colorizer(sde, sampling.ReverseDiffusionPredictor, sampling.LangevinCorrector, lambda v: v, **kw)
  torch.manual_seed(0)
  data = torch.rand(2, 3, 4, 4)
  inp(Zero(), data, (torch.rand(2, 1, 4, 4) > 0.5).float())
  assert inp.last_stats['loop'] == 'host'
  col(Zero(), data.mean(1, keepdim=True).expand(2, 3, 4, 4).contiguous())
  assert col.last_stats['loop'] == 'host'


def test_constrained_plan_rejects_an_unknown_constraint():
  with pytest.raises(ValueError, match='outpaint'):
    native.ConstrainedPcPlan(None, sde_lib.VESDE(0.01, 50, 3), 'reverse_diffusion', 'langevin', (1, 3, 4, 4), 0.16, 1,
                             False, 1e-5, 'cuda', constraint='outpaint')


@pytest.mark.parametrize('task,batch,layout', [('inpaint', 2, 'nchw'), ('colorize', 2, 'nhwc'), ('colorize', 1, 'nchw')])
def test_host_loop_draws_keep_the_initial_state_layout(monkeypatch, task, batch, layout):
  """torch.randn_like fills a dense tensor in memory order.  The native loop assumes every draw of the reference loop
  sees the layout of the initial state (channels-last for the colorizer's einsum output at batch > 1), for every stock
  predictor and corrector; this records the layout at each draw of the host loop."""
  from score_sde_pytorch_b200 import controllable_generation as CG, sampling

  class Const(torch.nn.Module):
    def forward(self, x, labels):
      return torch.full(x.shape, 0.1)

  seen, orig = [], torch.randn_like

  def spy(x, *a, **k):
    seen.append('nchw' if x.is_contiguous() else 'nhwc' if x.is_contiguous(memory_format=torch.channels_last) else '?')
    return orig(x, *a, **k)

  monkeypatch.setattr(torch, 'randn_like', spy)
  torch.manual_seed(0)
  data = torch.rand(batch, 3, 8, 8)
  sdes = [sde_lib.VESDE(0.01, 50, 4), sde_lib.VPSDE(0.1, 20., 30), sde_lib.subVPSDE(0.1, 20., 30)]
  preds = [sampling.ReverseDiffusionPredictor, sampling.EulerMaruyamaPredictor, sampling.AncestralSamplingPredictor,
           sampling.NonePredictor]
  corrs = [sampling.LangevinCorrector, sampling.AnnealedLangevinDynamics, sampling.NoneCorrector]
  runs = 0
  for sde in sdes:
    for P in preds:
      for C in corrs:
        if isinstance(sde, sde_lib.subVPSDE) and (P is sampling.AncestralSamplingPredictor or C is not sampling.NoneCorrector):
          continue   # the reference raises for these
        make = CG.get_pc_inpainter if task == 'inpaint' else CG.get_pc_colorizer
        fn = make(sde, P, C, lambda v: v, snr=0.16, n_steps=2, probability_flow=False, continuous=True)
        seen.clear()
        if task == 'inpaint':
          fn(Const(), data, (torch.rand(batch, 1, 8, 8) > 0.5).float())
        else:
          fn(Const(), data.mean(1, keepdim=True).expand(batch, 3, 8, 8).contiguous())
        assert seen and set(seen) == {layout}, (type(sde).__name__, P.__name__, C.__name__, set(seen))
        runs += 1
  assert runs == 27
