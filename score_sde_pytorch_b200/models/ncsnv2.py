"""NCSNv2 score networks backed by the sm_90a engine.

Host-side mirror of the reference's ``models/ncsnv2.py`` (``NCSNv2`` registered as ``'ncsnv2_64'``, ``NCSNv2_128`` as
``'ncsnv2_128'``), as configured by ``configs/ve/ncsnv2/*.py``: the modules carry the reference's names, shapes and
PyTorch default initialisers, so ``state_dict()`` / ``load_state_dict()`` interoperate with reference checkpoints
(``sigmas`` buffer included) and ``parameters()`` comes in the reference's order.

The forward runs on the engine (``b200_ncsnpp_config.family = 2``): ResidualBlocks with InstanceNorm2dPlus + ELU,
dilated 3x3 convolutions and ConvMeanPool, RefineBlocks (RCU, MSF, CRP with 5x5 max pooling), and the output divided
by ``sigmas[y]``.  ``y`` holds integer noise-level indices, as ``get_score_fn`` passes them for ``continuous=False``.
The engine computes in fp32 and divides by sigma in fp32; ``forward`` returns the result cast to ``sigmas.dtype``
(float64), the dtype the reference's ``output / used_sigmas`` has.
"""
import torch
import torch.nn as nn

from .. import _lib
from . import utils
from ._engine import EngineModel


class _INPlus(nn.Module):
  """``InstanceNorm2dPlus(C, bias=True)`` (``normalization.py:157-169``): alpha, gamma ~ N(1, 0.02), beta = 0."""

  def __init__(self, c):
    super().__init__()
    self.alpha = nn.Parameter(torch.zeros(c).normal_(1, 0.02))
    self.gamma = nn.Parameter(torch.zeros(c).normal_(1, 0.02))
    self.beta = nn.Parameter(torch.zeros(c))


def _conv3(cin, cout, bias=True, dilation=1):
  """``ncsn_conv3x3`` (``layers.py:108-115``, PyTorch default init); dilated filters pad by their dilation."""
  return nn.Conv2d(cin, cout, 3, padding=dilation, dilation=dilation, bias=bias)


class _Holder(nn.Module):
  pass


class _RCU(nn.Module):
  """``RCUBlock(features, n_blocks, 2)`` (``layers.py:183-204``): ``{i}_{j}_conv``, 3x3 without bias."""

  def __init__(self, c, n_blocks):
    super().__init__()
    for i in range(n_blocks):
      for j in range(2):
        setattr(self, f'{i + 1}_{j + 1}_conv', _conv3(c, c, bias=False))


def _residual_block(cin, cout, down, dilation):
  """``ResidualBlock`` (``layers.py:453-503``) in its registration order: conv1, normalize2, conv2, shortcut, normalize1."""
  h = _Holder()
  mid = cin if down else cout
  h.conv1 = _conv3(cin, mid, dilation=dilation)
  h.normalize2 = _INPlus(mid)
  if down and dilation == 1:   # ConvMeanPool (layers.py:351-369): the convolution sits in `.conv`
    h.conv2 = _Holder()
    h.conv2.conv = _conv3(mid, cout)
  else:
    h.conv2 = _conv3(mid, cout, dilation=dilation)
  if cout != cin or down:
    if dilation > 1:
      h.shortcut = _conv3(cin, cout, dilation=dilation)
    elif down:
      h.shortcut = _Holder()
      h.shortcut.conv = nn.Conv2d(cin, cout, 1)
    else:
      h.shortcut = nn.Conv2d(cin, cout, 1)   # ncsn_conv1x1
  h.normalize1 = _INPlus(cin)
  return h


def _refine_block(in_planes, features, start=False, end=False):
  """``RefineBlock`` (``layers.py:277-294``): adapt_convs, output_convs, msf (more than one input), crp."""
  h = _Holder()
  h.adapt_convs = nn.ModuleList([_RCU(c, 2) for c in in_planes])
  h.output_convs = _RCU(features, 3 if end else 1)
  if not start:
    h.msf = _Holder()
    h.msf.convs = nn.ModuleList([_conv3(c, features) for c in in_planes])
  h.crp = _Holder()
  h.crp.convs = nn.ModuleList([_conv3(features, features, bias=False) for _ in range(2)])
  return h


class _NCSNv2Base(EngineModel):
  """Shared constructor of the two NCSNv2 walks.  ``precision``: ``'tf32'`` (default), ``'f16'`` or ``'fp32'``; split
  TF32 (``'tf32x3'``) is not implemented for this family.  ``keep_activations=True`` records every block output for
  :meth:`tap` (indices: :meth:`tap_names`)."""
  LEVELS = None      # (output channels as multiples of nf, dilation) per level
  REFINE = None      # refine block output channels as multiples of nf
  SIZES = None       # image sizes the walk takes
  takes_time_labels = False   # y is an index into sigmas: the native PC loop, ODE solver and likelihood are not used

  def __init__(self, config, precision=None, keep_activations=False, lanes=1, pdl=None, halo=None):
    super().__init__()
    self.config = config
    m, name = config.model, type(self).__name__
    size = config.data.image_size
    if size == 28:
      raise NotImplementedError(f'{name}: data.image_size=28 (the adjust_padding blocks of models/ncsnv2.py:77-82) is not '
                                'supported by the engine')
    if not self.SIZES(size):
      raise NotImplementedError(f'{name}: data.image_size={size} is outside this network\'s walk on the engine')
    if m.normalization != 'InstanceNorm++':
      raise NotImplementedError(f"{name}: model.normalization={m.normalization!r}; the engine implements 'InstanceNorm++' only")
    if m.nonlinearity.lower() != 'elu':
      raise NotImplementedError(f"{name}: model.nonlinearity={m.nonlinearity!r}; the engine implements 'elu' only")
    if getattr(m, 'interpolation', 'bilinear') != 'bilinear':
      raise NotImplementedError(f"{name}: model.interpolation={m.interpolation!r}; the engine implements 'bilinear' only")
    self._set_engine_options(config, precision, keep_activations, lanes, None, pdl, halo)
    if self.precision == 'tf32x3':
      raise NotImplementedError(f"{name}: precision='tf32x3' is not implemented for NCSNv2; use 'tf32', 'f16' or 'fp32'")
    self.register_buffer('sigmas', torch.tensor(utils.get_sigmas(config)))   # fp64, as ncsnv2.py:51
    nf, ch = m.nf, config.data.num_channels
    self.begin_conv = nn.Conv2d(ch, nf, 3, padding=1)
    self.normalizer = _INPlus(nf)
    self.end_conv = nn.Conv2d(nf, ch, 3, padding=1)
    cin = nf
    for lvl, (mult, dil) in enumerate(self.LEVELS):
      cout = mult * nf
      blocks = [_residual_block(cin, cout, down=lvl > 0, dilation=dil), _residual_block(cout, cout, down=False, dilation=dil)]
      setattr(self, f'res{lvl + 1}', nn.ModuleList(blocks))
      cin = cout
    L = len(self.LEVELS)
    for k in range(1, L + 1):
      lay = self.LEVELS[L - k][0] * nf
      ins = [lay] if k == 1 else [lay, self.REFINE[k - 2] * nf]
      setattr(self, f'refine{k}', _refine_block(ins, self.REFINE[k - 1] * nf, start=k == 1, end=k == L))
    self._init_engine()

  def tap_names(self):
    """Module of each :meth:`tap` index: begin_conv, the ResidualBlocks, then the RefineBlocks, in forward order."""
    L = len(self.LEVELS)
    return (['begin_conv'] + [f'res{l + 1}.{b}' for l in range(L) for b in range(2)] +
            [f'refine{k}' for k in range(1, L + 1)])

  def _native_config(self):
    cfg = self.config
    c = _lib.NcsnppConfig()
    c.image_size, c.num_channels, c.nf = cfg.data.image_size, cfg.data.num_channels, cfg.model.nf
    c.num_levels = len(self.LEVELS)
    c.centered = int(bool(cfg.data.centered))
    c.scale_by_sigma, c.conditional, c.num_res_blocks = 1, 1, 2
    self._execution_config(c)
    c.family = 2
    return c

  def check_jvp_supported(self):
    raise NotImplementedError(f'{type(self).__name__}.jvp: NCSNv2 has no forward-mode tangent pass on the engine')

  def jvp(self, x, time_cond, v, labels_uniform=False):
    self.check_jvp_supported()

  def forward(self, x, y):
    """``output / sigmas[y]`` for integer noise-level indices ``y`` (``ncsnv2.py:107-132``)."""
    if torch.is_floating_point(y) or torch.is_complex(y):
      raise TypeError(f'{type(self).__name__}: y holds noise-level indices (an integer tensor, as get_score_fn passes for '
                      f'continuous=False), got {y.dtype}; continuous-time labels have no meaning for this network')
    sig = self.sigmas.to(x.device)[y.to(x.device).long()].to(torch.float32)
    out = super().forward(x, sig)
    return out.to(self.sigmas.dtype)


@utils.register_model(name='ncsnv2_64')
class NCSNv2(_NCSNv2Base):
  """``models/ncsnv2.py:43-132``: four levels (nf, 2nf, 2nf dilated 2, 2nf dilated 4), four RefineBlocks."""
  LEVELS = ((1, 1), (2, 1), (2, 2), (2, 4))
  REFINE = (2, 2, 1, 1)
  SIZES = staticmethod(lambda s: 16 <= s < 96 and s % 4 == 0)


@utils.register_model(name='ncsnv2_128')
class NCSNv2_128(_NCSNv2Base):
  """``models/ncsnv2.py:221-312``: five levels (nf, 2nf, 2nf, 4nf dilated 2, 4nf dilated 4), five RefineBlocks."""
  LEVELS = ((1, 1), (2, 1), (2, 1), (4, 2), (4, 4))
  REFINE = (4, 2, 2, 1, 1)
  SIZES = staticmethod(lambda s: 96 <= s <= 128 and s % 8 == 0)


def _refused(name, why):
  class _Refused:
    def __init__(self, config, *args, **kwargs):
      raise NotImplementedError(f"model.name={name!r}: {why}")
  _Refused.__name__ = f'Refused_{name}'
  return _Refused


utils.register_model(_refused('ncsnv2_256', 'NCSNv2_256 is not implemented on the engine (no reference config uses it)'),
                     name='ncsnv2_256')
utils.register_model(_refused('ncsn', 'NCSN v1 (conditional instance normalisation) is not implemented on the engine'),
                     name='ncsn')
