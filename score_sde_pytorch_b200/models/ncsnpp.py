"""NCSN++ score network backed by the sm_90a engine.

Host-side mirror of ``models/ncsnpp.py:35-381``: ``NCSNpp(config)`` is an
``nn.Module`` registered as ``'ncsnpp'``; its parameters live in
``all_modules`` with the reference's names, shapes and initialisers, so
``state_dict()`` / ``load_state_dict()`` interoperate with reference checkpoints
(with or without the ``module.`` prefix DataParallel adds, ``utils.py:16``), and
``forward(x[B,C,H,W], time_cond[B]) -> [B,C,H,W]`` has the reference's meaning.

The forward itself is not PyTorch: parameters are repacked once into the
engine's blob (K-major, TF32-rounded where a layer runs on the tensor cores) and every
call replays the engine's kernel sequence on the current CUDA stream through the
C ABI (``include/scoresde_b200.h``).  CPU tensors are rejected — there is no CPU
path in the product (the plain-PyTorch restatement lives in ``oracle/`` and is
test infrastructure only).
"""
import numpy as np
import torch
import torch.nn as nn

from . import utils
from ._engine import EngineModel, positional_frequencies

_SUPPORTED = ("engine supports embedding_type in {'fourier','positional'}, conditional=True, resblock_type='biggan', "
              "fir in {True, False} (progressive_input='residual' needs fir=True), progressive in {'none','output_skip'}, "
              "progressive_input in {'none','residual','input_skip'} with progressive_combine='sum'; "
              "positional embeddings need scale_by_sigma=False")


def _variance_scaling_uniform(shape, scale, in_axis=1, out_axis=0):
  """fan_avg / uniform variance scaling, the reference's ``default_init``
  (``models/layers.py:54-91``; ``scale == 0`` is replaced by ``1e-10`` there, ``:88-91``)."""
  scale = 1e-10 if scale == 0 else scale
  rf = np.prod(shape) / shape[in_axis] / shape[out_axis]
  denom = (shape[in_axis] * rf + shape[out_axis] * rf) / 2
  return (torch.rand(*shape, dtype=torch.float32) * 2. - 1.) * np.sqrt(3 * scale / denom)


class _Holder(nn.Module):
  """Parameter container; submodule / parameter names follow the reference."""


def _conv(cin, cout, k, init_scale=1.):
  m = nn.Conv2d(cin, cout, kernel_size=k, stride=1, padding=k // 2)
  m.weight.data = _variance_scaling_uniform(m.weight.shape, init_scale)
  nn.init.zeros_(m.bias)
  return m


def _gn(c):
  return nn.GroupNorm(num_groups=min(c // 4, 32), num_channels=c, eps=1e-6)


def _dense(cin, cout):
  m = nn.Linear(cin, cout)
  m.weight.data = _variance_scaling_uniform(m.weight.shape, 1.)
  nn.init.zeros_(m.bias)
  return m


class _NIN(nn.Module):
  def __init__(self, cin, cout, init_scale=0.1):
    super().__init__()
    self.W = nn.Parameter(_variance_scaling_uniform((cin, cout), init_scale))
    self.b = nn.Parameter(torch.zeros(cout))


class _Fourier(nn.Module):
  def __init__(self, size, scale):
    super().__init__()
    self.W = nn.Parameter(torch.randn(size) * scale, requires_grad=False)


def _resblock(cin, cout, temb_dim, init_scale, up=False, down=False):
  h = _Holder()
  h.GroupNorm_0 = _gn(cin)
  h.Conv_0 = _conv(cin, cout, 3)
  h.Dense_0 = _dense(temb_dim, cout)
  h.GroupNorm_1 = _gn(cout)
  h.Conv_1 = _conv(cout, cout, 3, init_scale)
  if cin != cout or up or down:
    h.Conv_2 = _conv(cin, cout, 1)
  return h


def _attn(c, init_scale):
  h = _Holder()
  h.GroupNorm_0 = _gn(c)
  h.NIN_0, h.NIN_1, h.NIN_2 = _NIN(c, c), _NIN(c, c), _NIN(c, c)
  h.NIN_3 = _NIN(c, c, init_scale=init_scale)
  return h


def _combine(dim1, dim2):
  """``layerspp.Combine`` (``layerspp.py:44-59``): ``Conv_0`` is a 1x1 convolution dim1 -> dim2."""
  h = _Holder()
  h.Conv_0 = _conv(dim1, dim2, 1)
  return h


def _pyramid_down(cin, cout):
  h = _Holder()
  inner = _Holder()
  inner.weight = nn.Parameter(_variance_scaling_uniform((cout, cin, 3, 3), 1.))
  inner.bias = nn.Parameter(torch.zeros(cout))
  h.Conv2d_0 = inner
  return h


@utils.register_model(name='ncsnpp')
class NCSNpp(EngineModel):
  """NCSN++ model (engine-backed).  ``precision``: ``'tf32'`` (wgmma tensor cores on TF32-rounded
  fp32 operands, default), ``'f16'`` (wgmma on fp16 operands: the same 11-bit significand as TF32
  with fp32 accumulation and fp32 activations between layers, half the operand traffic and twice the
  MMA rate), ``'tf32x3'`` (split TF32: hi + lo TF32 pairs, three wgmma products per K step; close to fp32
  accuracy on the tensor cores, about 3x the MMA work of ``'tf32'``) or ``'fp32'`` (strict fp32 on CUDA cores;
  validation mode).  The engine plumbing is
  ``models._engine.EngineModel``."""

  def __init__(self, config, precision=None, keep_activations=False, lanes=1, cuda_core_head=None, pdl=None,
               halo=None):
    super().__init__()
    self.config = config
    m = config.model
    emb = m.embedding_type.lower()
    if (emb not in ('fourier', 'positional') or not m.conditional or m.resblock_type.lower() != 'biggan'
        or m.progressive.lower() not in ('none', 'output_skip')
        or m.progressive_input.lower() not in ('none', 'residual', 'input_skip')
        or (m.progressive_input.lower() == 'input_skip' and str(getattr(m, 'progressive_combine', 'sum')).lower() != 'sum')
        or (not m.fir and m.progressive_input.lower() == 'residual')
        or (emb == 'positional' and m.scale_by_sigma)):
      raise NotImplementedError(f'NCSNpp: {_SUPPORTED}')
    if m.nonlinearity.lower() != 'swish':
      raise NotImplementedError('NCSNpp: engine implements the swish (SiLU) nonlinearity only')
    assert emb != 'fourier' or config.training.continuous, "Fourier features are only used for continuous training."
    self.register_buffer('sigmas', torch.tensor(utils.get_sigmas(config)))   # fp64, as ncsnpp.py:42
    self.embedding_type = emb
    self._set_engine_options(config, precision, keep_activations, lanes, cuda_core_head, pdl, halo)
    nf, ch_mult, nrb = m.nf, tuple(m.ch_mult), m.num_res_blocks
    L = len(ch_mult)
    all_res = [config.data.image_size // (2 ** i) for i in range(L)]
    channels = config.data.num_channels
    init_scale = m.init_scale
    temb_dim = nf * 4
    if emb == 'fourier':
      mods = [_Fourier(nf, m.fourier_scale), _dense(2 * nf, temb_dim), _dense(temb_dim, temb_dim)]
    else:
      # Sinusoidal embedding of the time label (models/layers.py:515-529): no parameters.  The frequency table is
      # built with the reference's own torch ops (so the engine multiplies by bit-identical fp32 frequencies) and kept
      # as a non-persistent buffer: it is not a state_dict key of the reference.
      mods = [_dense(nf, temb_dim), _dense(temb_dim, temb_dim)]
      half = nf // 2
      if nf % 2 or half < 2:
        raise NotImplementedError('NCSNpp: positional embedding needs an even nf >= 4')
      self.register_buffer('pos_freqs', positional_frequencies(nf), persistent=False)
    mods.append(_conv(channels, nf, 3))
    hs_c = [nf]
    in_ch, pyr_ch = nf, channels
    for lvl in range(L):
      for _ in range(nrb):
        out_ch = nf * ch_mult[lvl]
        mods.append(_resblock(in_ch, out_ch, temb_dim, init_scale))
        in_ch = out_ch
        if all_res[lvl] in m.attn_resolutions:
          mods.append(_attn(in_ch, init_scale))
        hs_c.append(in_ch)
      if lvl != L - 1:
        mods.append(_resblock(in_ch, in_ch, temb_dim, init_scale, down=True))
        if m.progressive_input.lower() == 'input_skip':
          mods.append(_combine(channels, in_ch))
        elif m.progressive_input.lower() == 'residual':
          mods.append(_pyramid_down(pyr_ch, in_ch))
          pyr_ch = in_ch
        hs_c.append(in_ch)
    in_ch = hs_c[-1]
    mods += [_resblock(in_ch, in_ch, temb_dim, init_scale), _attn(in_ch, init_scale),
             _resblock(in_ch, in_ch, temb_dim, init_scale)]
    for lvl in reversed(range(L)):
      for _ in range(nrb + 1):
        out_ch = nf * ch_mult[lvl]
        mods.append(_resblock(in_ch + hs_c.pop(), out_ch, temb_dim, init_scale))
        in_ch = out_ch
      if all_res[lvl] in m.attn_resolutions:
        mods.append(_attn(in_ch, init_scale))
      if m.progressive.lower() == 'output_skip':      # ncsnpp.py:190-203
        mods.append(_gn(in_ch))
        mods.append(_conv(in_ch, channels, 3, init_scale))
      if lvl != 0:
        mods.append(_resblock(in_ch, in_ch, temb_dim, init_scale, up=True))
    assert not hs_c
    if m.progressive.lower() != 'output_skip':
      mods.append(_gn(in_ch))
      mods.append(_conv(in_ch, channels, 3, init_scale))
    self.all_modules = nn.ModuleList(mods)
    self._init_engine()

  def _family_config(self, c):
    m = self.config.model
    c.family = 0
    c.skip_rescale = int(bool(m.skip_rescale))
    c.progressive_input = {'none': 0, 'residual': 1, 'input_skip': 2}[m.progressive_input.lower()]
    c.progressive = 1 if m.progressive.lower() == 'output_skip' else 0
    c.fir_taps = len(m.fir_kernel)
    for i, v in enumerate(m.fir_kernel):
      c.fir_kernel[i] = float(v)
    c.embedding_type = 1 if self.embedding_type == 'positional' else 0
    c.naive_resample = 0 if m.fir else 1
