"""DDPM score network backed by the sm_90a engine.

Host-side mirror of ``models/ddpm.py:39-181`` (the network of Ho et al., as configured by
``configs/vp/ddpm/*.py`` and ``configs/subvp/cifar10_ddpm_continuous.py``): ``DDPM(config)`` is an
``nn.Module`` registered as ``'ddpm'`` whose ``all_modules`` carry the reference's names, shapes and
initialisers, so ``state_dict()`` / ``load_state_dict()`` interoperate with reference checkpoints and
``parameters()`` comes in the reference's order (EMA shadow lists are positional).

The forward runs on the same engine as ``NCSNpp`` (``b200_ncsnpp_config.family = 1``): ResnetBlockDDPM
(``layers.py:619-662``) with its ``NIN_0`` skip fused into the second convolution, AttnBlock
(``:558-581``), Downsample / Upsample with_conv (``:584-616``), GroupNorm with 32 groups and residual
scale 1 throughout, sinusoidal time embedding (``layers.py:515-529``).
"""
import torch
import torch.nn as nn

from . import utils
from ._engine import EngineModel, positional_frequencies
from .ncsnpp import _Holder, _NIN, _conv, _dense


def _gn(c):
  return nn.GroupNorm(num_groups=32, num_channels=c, eps=1e-6)


def _resblock(cin, cout, temb_dim):
  """``ResnetBlockDDPM(act, in_ch, out_ch, temb_dim)`` (``layers.py:619-643``); Dropout_0 has no parameters."""
  h = _Holder()
  h.GroupNorm_0 = _gn(cin)
  h.Conv_0 = _conv(cin, cout, 3)
  h.Dense_0 = _dense(temb_dim, cout)
  h.GroupNorm_1 = _gn(cout)
  h.Conv_1 = _conv(cout, cout, 3, init_scale=0.)
  if cin != cout:
    h.NIN_0 = _NIN(cin, cout)
  return h


def _attn(c):
  """``AttnBlock(channels)`` (``layers.py:558-566``)."""
  h = _Holder()
  h.GroupNorm_0 = _gn(c)
  h.NIN_0, h.NIN_1, h.NIN_2 = _NIN(c, c), _NIN(c, c), _NIN(c, c)
  h.NIN_3 = _NIN(c, c, init_scale=0.)
  return h


def _resample(c, down):
  """``Downsample`` / ``Upsample`` with ``with_conv=True`` (``layers.py:584-605``): one 3x3 ``Conv_0``, C -> C."""
  h = _Holder()
  h.Conv_0 = _conv(c, c, 3)
  if down:   # stride 2, no padding: the (0,1,0,1) pad is explicit in the reference's forward
    h.Conv_0.stride, h.Conv_0.padding = (2, 2), (0, 0)
  return h


@utils.register_model(name='ddpm')
class DDPM(EngineModel):
  """DDPM model (engine-backed).  Same execution options as ``NCSNpp``: ``precision`` in ``'tf32'`` (default),
  ``'f16'``, ``'tf32x3'`` (split TF32, close to fp32 accuracy on the tensor cores), ``'fp32'``; ``keep_activations`` (debug taps), ``lanes``, ``pdl``."""

  def __init__(self, config, precision=None, keep_activations=False, lanes=1, cuda_core_head=None, pdl=None,
               halo=None):
    super().__init__()
    self.config = config
    m = config.model
    if not m.conditional:
      raise NotImplementedError('DDPM: conditional=False is not supported (the reference constructor itself fails '
                                'without time conditioning, models/ddpm.py:58-71)')
    if m.scale_by_sigma:
      raise NotImplementedError('DDPM: scale_by_sigma=True (configs/ve/cifar10_ddpm.py) is not supported by the engine')
    if not m.resamp_with_conv:
      raise NotImplementedError('DDPM: resamp_with_conv=False is not supported by the engine')
    if m.nonlinearity.lower() != 'swish':
      raise NotImplementedError('DDPM: engine implements the swish (SiLU) nonlinearity only')
    self.register_buffer('sigmas', torch.tensor(utils.get_sigmas(config)))   # fp64, as ddpm.py:44
    self._set_engine_options(config, precision, keep_activations, lanes, cuda_core_head, pdl, halo)
    nf, ch_mult, nrb = m.nf, tuple(m.ch_mult), m.num_res_blocks
    if nf % 2 or nf < 4:
      raise NotImplementedError('DDPM: the sinusoidal time embedding needs an even nf >= 4')
    # frequency table of the time embedding (ddpm.py:116): a non-persistent buffer, not a state_dict key of the reference
    self.register_buffer('pos_freqs', positional_frequencies(nf), persistent=False)
    L = len(ch_mult)
    all_res = [config.data.image_size // (2 ** i) for i in range(L)]
    channels = config.data.num_channels
    temb_dim = 4 * nf
    mods = [_dense(nf, temb_dim), _dense(temb_dim, temb_dim), _conv(channels, nf, 3)]
    hs_c = [nf]
    in_ch = nf
    for lvl in range(L):
      for _ in range(nrb):
        out_ch = nf * ch_mult[lvl]
        mods.append(_resblock(in_ch, out_ch, temb_dim))
        in_ch = out_ch
        if all_res[lvl] in m.attn_resolutions:
          mods.append(_attn(in_ch))
        hs_c.append(in_ch)
      if lvl != L - 1:
        mods.append(_resample(in_ch, down=True))
        hs_c.append(in_ch)
    in_ch = hs_c[-1]
    mods += [_resblock(in_ch, in_ch, temb_dim), _attn(in_ch), _resblock(in_ch, in_ch, temb_dim)]
    for lvl in reversed(range(L)):
      for _ in range(nrb + 1):
        out_ch = nf * ch_mult[lvl]
        mods.append(_resblock(in_ch + hs_c.pop(), out_ch, temb_dim))
        in_ch = out_ch
      if all_res[lvl] in m.attn_resolutions:
        mods.append(_attn(in_ch))
      if lvl != 0:
        mods.append(_resample(in_ch, down=False))
    assert not hs_c
    mods += [_gn(in_ch), _conv(in_ch, channels, 3, init_scale=0.)]
    self.all_modules = nn.ModuleList(mods)
    self._init_engine()

  def _family_config(self, c):
    c.family = 1
