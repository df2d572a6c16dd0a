"""ORACLE (test infrastructure, not product code): plain PyTorch fp32 restatement
of the reference's NCSN++ score network.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import this module.  The product path
(``score_sde_pytorch_b200``) never does; it fails loudly without its CUDA library.

Pinning: ``tools/make_golden.py`` runs the *real* reference
(``/root/reference/models/ncsnpp.py`` imported in the build container) on seeded
inputs with weights loaded from the same ``state_dict`` and commits small
fixtures under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this
file against them.  The ``state_dict`` key names are the reference's
(``all_modules.{i}.…``), so a reference checkpoint loads
unchanged.

Each function cites the reference lines it follows.  The arithmetic is written
with ordinary torch ops (``F.conv2d``, ``F.group_norm``, ``torch.einsum`` …) in
the reference's operation order, in NCHW, so that on CPU it is bit-comparable
with the reference's own CPU path.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

SQRT2 = np.sqrt(2.)


# ----------------------------------------------------------------------------
# FIR resampling  (op/upfirdn2d.py:159-200, models/up_or_down_sampling.py)
# ----------------------------------------------------------------------------
def upfirdn2d_native(x, kernel, up=1, down=1, pad=(0, 0)):
  """Zero-insert upsample, pad, correlate with the flipped FIR, decimate.
  Follows ``upfirdn2d_native`` (op/upfirdn2d.py:159-200) for an NCHW tensor with
  symmetric (x == y) up/down/pad as ``upfirdn2d`` passes them (``:145-156``)."""
  n, c, in_h, in_w = x.shape
  kh, kw = kernel.shape
  p0, p1 = pad
  v = x.reshape(-1, in_h, 1, in_w, 1, 1)
  v = F.pad(v, [0, 0, 0, up - 1, 0, 0, 0, up - 1])
  v = v.view(-1, in_h * up, in_w * up, 1)
  v = F.pad(v, [0, 0, max(p0, 0), max(p1, 0), max(p0, 0), max(p1, 0)])
  v = v[:, max(-p0, 0): v.shape[1] - max(-p1, 0), max(-p0, 0): v.shape[2] - max(-p1, 0), :]
  v = v.permute(0, 3, 1, 2).reshape(-1, 1, in_h * up + p0 + p1, in_w * up + p0 + p1)
  w = torch.flip(kernel, [0, 1]).view(1, 1, kh, kw)
  v = F.conv2d(v, w)
  v = v.reshape(-1, 1, in_h * up + p0 + p1 - kh + 1, in_w * up + p0 + p1 - kw + 1)
  v = v.permute(0, 2, 3, 1)[:, ::down, ::down, :]
  out_h = (in_h * up + p0 + p1 - kh) // down + 1
  out_w = (in_w * up + p0 + p1 - kw) // down + 1
  return v.reshape(n, c, out_h, out_w)


def setup_kernel(k):
  """Separable taps -> normalised 2-D fp32 FIR (up_or_down_sampling.py:181-188)."""
  k = np.asarray(k, dtype=np.float32)
  if k.ndim == 1:
    k = np.outer(k, k)
  k /= np.sum(k)
  return k


def upsample_2d(x, k, factor=2, gain=1):
  """up_or_down_sampling.py:195-224."""
  k = setup_kernel(k) * (gain * (factor ** 2))
  p = k.shape[0] - factor
  return upfirdn2d_native(x, torch.tensor(k, device=x.device), up=factor,
                          pad=((p + 1) // 2 + factor - 1, p // 2))


def downsample_2d(x, k, factor=2, gain=1):
  """up_or_down_sampling.py:227-257."""
  k = setup_kernel(k) * gain
  p = k.shape[0] - factor
  return upfirdn2d_native(x, torch.tensor(k, device=x.device), down=factor,
                          pad=((p + 1) // 2, p // 2))


def conv_downsample_2d(x, w, k, factor=2, gain=1):
  """FIR pad-filter then stride-``factor`` VALID conv (up_or_down_sampling.py:144-178)."""
  conv_w = w.shape[3]
  k = setup_kernel(k) * gain
  p = (k.shape[0] - factor) + (conv_w - 1)
  x = upfirdn2d_native(x, torch.tensor(k, device=x.device), pad=((p + 1) // 2, p // 2))
  return F.conv2d(x, w, stride=factor, padding=0)


def naive_upsample_2d(x, factor=2):
  """up_or_down_sampling.py:59-63."""
  n, c, h, w = x.shape
  x = x.reshape(-1, c, h, 1, w, 1).repeat(1, 1, 1, factor, 1, factor)
  return x.reshape(-1, c, h * factor, w * factor)


def naive_downsample_2d(x, factor=2):
  """up_or_down_sampling.py:66-69."""
  n, c, h, w = x.shape
  return torch.mean(x.reshape(-1, c, h // factor, factor, w // factor, factor), dim=(3, 5))


def fused_leaky_relu(x, bias, negative_slope=0.2, scale=2 ** 0.5):
  """CPU branch of op/fused_act.py:86-94 (note: the reference hard-codes 0.2 there)."""
  rest = [1] * (x.ndim - bias.ndim - 1)
  return F.leaky_relu(x + bias.view(1, bias.shape[0], *rest), negative_slope=0.2) * scale


# ----------------------------------------------------------------------------
# Graph description: the same walk as NCSNpp.__init__ (models/ncsnpp.py:68-230)
# ----------------------------------------------------------------------------
def build_module_specs(config):
  """List of dicts, one per ``all_modules`` entry, in construction order."""
  m = config.model
  nf, ch_mult, nrb = m.nf, tuple(m.ch_mult), m.num_res_blocks
  num_res = len(ch_mult)
  all_res = [config.data.image_size // (2 ** i) for i in range(num_res)]
  resblock_type = m.resblock_type.lower()
  progressive = m.progressive.lower()
  progressive_input = m.progressive_input.lower()
  combine = m.progressive_combine.lower()
  channels = config.data.num_channels
  specs = []

  def add(kind, **kw):
    specs.append(dict(kind=kind, **kw))

  if m.embedding_type.lower() == 'fourier':
    add('fourier', size=nf)
    embed_dim = 2 * nf
  else:
    embed_dim = nf
  if m.conditional:
    add('linear', cin=embed_dim, cout=nf * 4)
    add('linear', cin=nf * 4, cout=nf * 4)

  def resblock(cin, cout=None, up=False, down=False):
    cout = cout if cout else cin
    if resblock_type == 'biggan':
      add('resblock_biggan', cin=cin, cout=cout, up=up, down=down)
    else:
      add('resblock_ddpm', cin=cin, cout=cout)

  input_pyramid_ch = channels
  add('conv3x3', cin=channels, cout=nf)
  hs_c = [nf]
  in_ch = nf
  for lvl in range(num_res):
    for _ in range(nrb):
      out_ch = nf * ch_mult[lvl]
      resblock(in_ch, out_ch)
      in_ch = out_ch
      if all_res[lvl] in m.attn_resolutions:
        add('attn', c=in_ch)
      hs_c.append(in_ch)
    if lvl != num_res - 1:
      if resblock_type == 'ddpm':
        add('downsample', cin=in_ch, cout=in_ch, with_conv=m.resamp_with_conv)
      else:
        resblock(in_ch, down=True)
      if progressive_input == 'input_skip':
        add('combine', dim1=input_pyramid_ch, dim2=in_ch, method=combine)
        if combine == 'cat':
          in_ch *= 2
      elif progressive_input == 'residual':
        add('downsample', cin=input_pyramid_ch, cout=in_ch, with_conv=True)
        input_pyramid_ch = in_ch
      hs_c.append(in_ch)

  in_ch = hs_c[-1]
  resblock(in_ch)
  add('attn', c=in_ch)
  resblock(in_ch)

  pyramid_ch = 0
  for lvl in reversed(range(num_res)):
    for _ in range(nrb + 1):
      out_ch = nf * ch_mult[lvl]
      resblock(in_ch + hs_c.pop(), out_ch)
      in_ch = out_ch
    if all_res[lvl] in m.attn_resolutions:
      add('attn', c=in_ch)
    if progressive != 'none':
      if lvl == num_res - 1:
        add('groupnorm', c=in_ch)
        if progressive == 'output_skip':
          add('conv3x3', cin=in_ch, cout=channels)
          pyramid_ch = channels
        else:
          add('conv3x3', cin=in_ch, cout=in_ch)
          pyramid_ch = in_ch
      else:
        if progressive == 'output_skip':
          add('groupnorm', c=in_ch)
          add('conv3x3', cin=in_ch, cout=channels)
          pyramid_ch = channels
        else:
          add('upsample', cin=pyramid_ch, cout=in_ch, with_conv=True)
          pyramid_ch = in_ch
    if lvl != 0:
      if resblock_type == 'ddpm':
        add('upsample', cin=in_ch, cout=in_ch, with_conv=m.resamp_with_conv)
      else:
        resblock(in_ch, up=True)
  assert not hs_c
  if progressive != 'output_skip':
    add('groupnorm', c=in_ch)
    add('conv3x3', cin=in_ch, cout=channels)
  return specs


# ----------------------------------------------------------------------------
# Blocks
# ----------------------------------------------------------------------------
def _gn(x, p, prefix):
  c = x.shape[1]
  return F.group_norm(x, min(c // 4, 32), p[prefix + '.weight'], p[prefix + '.bias'], eps=1e-6)


def _conv(x, p, prefix, padding):
  return F.conv2d(x, p[prefix + '.weight'], p[prefix + '.bias'], stride=1, padding=padding)


def _nin(x, p, prefix):
  """layers.py:546-555: per-pixel ``x·W + b`` with ``W[in,out]``."""
  y = torch.einsum('bhwc,cd->bhwd', x.permute(0, 2, 3, 1), p[prefix + '.W']) + p[prefix + '.b']
  return y.permute(0, 3, 1, 2)


def resblock_biggan(x, temb, p, pre, spec, cfg):
  """layerspp.py:242-274."""
  m = cfg.model
  h = F.silu(_gn(x, p, pre + '.GroupNorm_0'))
  if spec['up']:
    if m.fir:
      h, x = upsample_2d(h, m.fir_kernel), upsample_2d(x, m.fir_kernel)
    else:
      h, x = naive_upsample_2d(h), naive_upsample_2d(x)
  elif spec['down']:
    if m.fir:
      h, x = downsample_2d(h, m.fir_kernel), downsample_2d(x, m.fir_kernel)
    else:
      h, x = naive_downsample_2d(h), naive_downsample_2d(x)
  h = _conv(h, p, pre + '.Conv_0', 1)
  if temb is not None:
    h = h + F.linear(F.silu(temb), p[pre + '.Dense_0.weight'], p[pre + '.Dense_0.bias'])[:, :, None, None]
  h = F.silu(_gn(h, p, pre + '.GroupNorm_1'))
  h = _conv(h, p, pre + '.Conv_1', 1)          # dropout is inert in eval (models/utils.py:119-121)
  if spec['cin'] != spec['cout'] or spec['up'] or spec['down']:
    x = _conv(x, p, pre + '.Conv_2', 0)
  return (x + h) / SQRT2 if m.skip_rescale else x + h


def resblock_ddpm(x, temb, p, pre, spec, cfg):
  """layerspp.py:193-209."""
  h = F.silu(_gn(x, p, pre + '.GroupNorm_0'))
  h = _conv(h, p, pre + '.Conv_0', 1)
  if temb is not None:
    h = h + F.linear(F.silu(temb), p[pre + '.Dense_0.weight'], p[pre + '.Dense_0.bias'])[:, :, None, None]
  h = F.silu(_gn(h, p, pre + '.GroupNorm_1'))
  h = _conv(h, p, pre + '.Conv_1', 1)
  if spec['cin'] != spec['cout']:
    x = _nin(x, p, pre + '.NIN_0')
  return (x + h) / SQRT2 if cfg.model.skip_rescale else x + h


def attn_block(x, p, pre, cfg):
  """layerspp.py:75-91."""
  b, c, hh, ww = x.shape
  h = _gn(x, p, pre + '.GroupNorm_0')
  q, k, v = _nin(h, p, pre + '.NIN_0'), _nin(h, p, pre + '.NIN_1'), _nin(h, p, pre + '.NIN_2')
  w = torch.einsum('bchw,bcij->bhwij', q, k) * (int(c) ** (-0.5))
  w = F.softmax(w.reshape(b, hh, ww, hh * ww), dim=-1).reshape(b, hh, ww, hh, ww)
  h = torch.einsum('bhwij,bcij->bchw', w, v)
  h = _nin(h, p, pre + '.NIN_3')
  return (x + h) / SQRT2 if cfg.model.skip_rescale else x + h


def downsample(x, p, pre, spec, cfg):
  """layerspp.py:148-163 / up_or_down_sampling.Conv2d.forward :44-56."""
  m = cfg.model
  if not m.fir:
    if spec['with_conv']:
      return F.conv2d(F.pad(x, (0, 1, 0, 1)), p[pre + '.Conv_0.weight'], p[pre + '.Conv_0.bias'], stride=2)
    return F.avg_pool2d(x, 2, stride=2)
  if not spec['with_conv']:
    return downsample_2d(x, m.fir_kernel)
  y = conv_downsample_2d(x, p[pre + '.Conv2d_0.weight'], m.fir_kernel)
  return y + p[pre + '.Conv2d_0.bias'].reshape(1, -1, 1, 1)


def upsample(x, p, pre, spec, cfg):
  """layerspp.py:113-126 (the fir+with_conv branch is dead in the reference:
  up_or_down_sampling.py:126 uses a negative-step slice torch rejects)."""
  m = cfg.model
  if not m.fir:
    h = F.interpolate(x, (x.shape[2] * 2, x.shape[3] * 2), mode='nearest')
    if spec['with_conv']:
      h = _conv(h, p, pre + '.Conv_0', 1)
    return h
  if not spec['with_conv']:
    return upsample_2d(x, m.fir_kernel)
  raise NotImplementedError('upsample_conv_2d is unreachable in the reference (negative-step slice)')


def timestep_embedding(timesteps, dim, max_positions=10000):
  """layers.py:515-529."""
  half = dim // 2
  e = math.log(max_positions) / (half - 1)
  e = torch.exp(torch.arange(half, dtype=torch.float32, device=timesteps.device) * -e)
  e = timesteps.float()[:, None] * e[None, :]
  e = torch.cat([torch.sin(e), torch.cos(e)], dim=1)
  if dim % 2 == 1:
    e = F.pad(e, (0, 1), mode='constant')
  return e


# ----------------------------------------------------------------------------
# Forward  (models/ncsnpp.py:232-381)
# ----------------------------------------------------------------------------
def ncsnpp_forward(params, config, x, time_cond, taps=None):
  """Score-network output for ``x[B,C,H,W]`` and ``time_cond[B]``.

  ``params``: dict of tensors keyed like the reference ``state_dict`` (a leading
  ``module.`` is accepted).  ``taps``: optional dict that receives the output of
  every ``all_modules`` entry by index (debug aid for per-layer parity tests).
  """
  p = {(k[7:] if k.startswith('module.') else k): v for k, v in params.items()}
  m = config.model
  specs = build_module_specs(config)
  num_res = len(m.ch_mult)
  attn_res = tuple(m.attn_resolutions)
  progressive = m.progressive.lower()
  progressive_input = m.progressive_input.lower()
  resblock_type = m.resblock_type.lower()
  i = 0

  def name(j):
    return f'all_modules.{j}'

  def tap(j, v):
    if taps is not None:
      taps[j] = v
    return v

  def run_resblock(h, temb):
    nonlocal i
    s = specs[i]
    fn = resblock_biggan if s['kind'] == 'resblock_biggan' else resblock_ddpm
    out = tap(i, fn(h, temb, p, name(i), s, config))
    i += 1
    return out

  def run_attn(h):
    nonlocal i
    out = tap(i, attn_block(h, p, name(i), config))
    i += 1
    return out

  if m.embedding_type.lower() == 'fourier':
    used_sigmas = time_cond
    proj = torch.log(used_sigmas)[:, None] * p[name(i) + '.W'][None, :] * 2 * np.pi   # layerspp.py:40
    temb = torch.cat([torch.sin(proj), torch.cos(proj)], dim=-1)
    i += 1
  else:
    used_sigmas = p['sigmas'][time_cond.long()]
    temb = timestep_embedding(time_cond, m.nf)
  if m.conditional:
    temb = F.linear(temb, p[name(i) + '.weight'], p[name(i) + '.bias']); i += 1
    temb = F.linear(F.silu(temb), p[name(i) + '.weight'], p[name(i) + '.bias']); i += 1
  else:
    temb = None

  if not config.data.centered:
    x = 2 * x - 1.
  input_pyramid = x if progressive_input != 'none' else None

  hs = [tap(i, _conv(x, p, name(i), 1))]
  i += 1
  for lvl in range(num_res):
    for _ in range(m.num_res_blocks):
      h = run_resblock(hs[-1], temb)
      if h.shape[-1] in attn_res:
        h = run_attn(h)
      hs.append(h)
    if lvl != num_res - 1:
      if resblock_type == 'ddpm':
        h = tap(i, downsample(hs[-1], p, name(i), specs[i], config)); i += 1
      else:
        h = run_resblock(hs[-1], temb)
      if progressive_input == 'input_skip':
        input_pyramid = downsample_2d(input_pyramid, m.fir_kernel) if m.fir else F.avg_pool2d(input_pyramid, 2, 2)
        y = _conv(input_pyramid, p, name(i) + '.Conv_0', 0)
        h = torch.cat([y, h], dim=1) if specs[i]['method'] == 'cat' else y + h
        tap(i, h); i += 1
      elif progressive_input == 'residual':
        input_pyramid = tap(i, downsample(input_pyramid, p, name(i), specs[i], config)); i += 1
        input_pyramid = (input_pyramid + h) / SQRT2 if m.skip_rescale else input_pyramid + h
        h = input_pyramid
      hs.append(h)

  h = hs[-1]
  h = run_resblock(h, temb)
  h = run_attn(h)
  h = run_resblock(h, temb)

  pyramid = None
  for lvl in reversed(range(num_res)):
    for _ in range(m.num_res_blocks + 1):
      h = run_resblock(torch.cat([h, hs.pop()], dim=1), temb)
    if h.shape[-1] in attn_res:
      h = run_attn(h)
    if progressive != 'none':
      if lvl == num_res - 1:
        pyramid = F.silu(_gn(h, p, name(i))); i += 1
        pyramid = _conv(pyramid, p, name(i), 1); i += 1
      elif progressive == 'output_skip':
        pyramid = upsample_2d(pyramid, m.fir_kernel) if m.fir else F.interpolate(pyramid, scale_factor=2, mode='nearest')
        ph = F.silu(_gn(h, p, name(i))); i += 1
        ph = _conv(ph, p, name(i), 1); i += 1
        pyramid = pyramid + ph
      else:
        pyramid = upsample(pyramid, p, name(i), specs[i], config); i += 1
        pyramid = (pyramid + h) / SQRT2 if m.skip_rescale else pyramid + h
        h = pyramid
    if lvl != 0:
      if resblock_type == 'ddpm':
        h = tap(i, upsample(h, p, name(i), specs[i], config)); i += 1
      else:
        h = run_resblock(h, temb)
  assert not hs

  if progressive == 'output_skip':
    h = pyramid
  else:
    h = F.silu(tap(i, _gn(h, p, name(i)))); i += 1
    h = tap(i, _conv(h, p, name(i), 1)); i += 1
  assert i == len(specs), (i, len(specs))
  if m.scale_by_sigma:
    h = h / used_sigmas.reshape((x.shape[0],) + (1,) * (x.dim() - 1))
  return h
