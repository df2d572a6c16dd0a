"""ORACLE (test infrastructure, not product code): plain PyTorch fp32 restatement of the
reference's DDPM score network (``models/ddpm.py:39-181`` with ``layers.py:558-662``).

Same rules as ``ncsnpp_oracle``: only tests, tools and benchmarks import it; ordinary torch ops in
the reference's operation order, NCHW, so that on CPU it is bit-comparable with the reference.  It is
pinned against fixtures written by the real reference (``tools/make_golden_ddpm.py``).
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.ncsnpp_oracle import _conv, _nin, timestep_embedding


def _gn(x, p, prefix):
  """Every DDPM GroupNorm has 32 groups (layers.py:562, 625, 633; ddpm.py:104)."""
  return F.group_norm(x, 32, p[prefix + '.weight'], p[prefix + '.bias'], eps=1e-6)


def resblock(x, temb, p, pre):
  """ResnetBlockDDPM.forward (layers.py:645-662); dropout is inert in eval."""
  h = F.silu(_gn(x, p, pre + '.GroupNorm_0'))
  h = _conv(h, p, pre + '.Conv_0', 1)
  h = h + F.linear(F.silu(temb), p[pre + '.Dense_0.weight'], p[pre + '.Dense_0.bias'])[:, :, None, None]
  h = F.silu(_gn(h, p, pre + '.GroupNorm_1'))
  h = _conv(h, p, pre + '.Conv_1', 1)
  if (pre + '.NIN_0.W') in p:
    x = _nin(x, p, pre + '.NIN_0')
  return x + h


def attn_block(x, p, pre):
  """AttnBlock.forward (layers.py:568-581)."""
  b, c, hh, ww = x.shape
  h = _gn(x, p, pre + '.GroupNorm_0')
  q, k, v = _nin(h, p, pre + '.NIN_0'), _nin(h, p, pre + '.NIN_1'), _nin(h, p, pre + '.NIN_2')
  w = torch.einsum('bchw,bcij->bhwij', q, k) * (int(c) ** (-0.5))
  w = F.softmax(w.reshape(b, hh, ww, hh * ww), dim=-1).reshape(b, hh, ww, hh, ww)
  h = torch.einsum('bhwij,bcij->bchw', w, v)
  return x + _nin(h, p, pre + '.NIN_3')


def downsample(x, p, pre):
  """Downsample(with_conv=True).forward (layers.py:606-616): pad (0,1,0,1), 3x3 stride-2 VALID conv."""
  return F.conv2d(F.pad(x, (0, 1, 0, 1)), p[pre + '.Conv_0.weight'], p[pre + '.Conv_0.bias'], stride=2)


def upsample(x, p, pre):
  """Upsample(with_conv=True).forward (layers.py:591-596)."""
  h = F.interpolate(x, (x.shape[2] * 2, x.shape[3] * 2), mode='nearest')
  return _conv(h, p, pre + '.Conv_0', 1)


def ddpm_forward(params, config, x, labels, taps=None):
  """DDPM.forward (models/ddpm.py:110-181) for ``x[B,C,H,W]`` and time labels ``labels[B]``.

  ``params``: tensors keyed like the reference ``state_dict`` (a leading ``module.`` is accepted).  ``taps``: optional
  dict receiving the output of every ``all_modules`` entry by index."""
  p = {(k[7:] if k.startswith('module.') else k): v for k, v in params.items()}
  m = config.model
  assert m.conditional and not m.scale_by_sigma and m.resamp_with_conv
  num_res = len(m.ch_mult)
  attn_res = tuple(m.attn_resolutions)
  i = 0

  def name(j):
    return f'all_modules.{j}'

  def tap(v):
    nonlocal i
    if taps is not None:
      taps[i] = v
    i += 1
    return v

  temb = timestep_embedding(labels, m.nf)
  temb = tap(F.linear(temb, p[name(i) + '.weight'], p[name(i) + '.bias']))
  temb = tap(F.linear(F.silu(temb), p[name(i) + '.weight'], p[name(i) + '.bias']))
  h = x if config.data.centered else 2 * x - 1.

  hs = [tap(_conv(h, p, name(i), 1))]
  for lvl in range(num_res):
    for _ in range(m.num_res_blocks):
      h = tap(resblock(hs[-1], temb, p, name(i)))
      if h.shape[-1] in attn_res:
        h = tap(attn_block(h, p, name(i)))
      hs.append(h)
    if lvl != num_res - 1:
      hs.append(tap(downsample(hs[-1], p, name(i))))

  h = hs[-1]
  h = tap(resblock(h, temb, p, name(i)))
  h = tap(attn_block(h, p, name(i)))
  h = tap(resblock(h, temb, p, name(i)))
  for lvl in reversed(range(num_res)):
    for _ in range(m.num_res_blocks + 1):
      h = tap(resblock(torch.cat([h, hs.pop()], dim=1), temb, p, name(i)))
    if h.shape[-1] in attn_res:
      h = tap(attn_block(h, p, name(i)))
    if lvl != 0:
      h = tap(upsample(h, p, name(i)))
  assert not hs
  h = F.silu(tap(_gn(h, p, name(i))))
  h = tap(_conv(h, p, name(i), 1))
  return h


def zero_init_keys(state_dict):
  """The weights the reference initialises with ``init_scale=0`` (variance scaling at 1e-10): ``Conv_1`` of every
  ResnetBlockDDPM, ``NIN_3`` of every AttnBlock and the output convolution (layers.py:566, 635; ddpm.py:105)."""
  last = max(int(k.split('.')[1]) for k in state_dict if k.startswith('all_modules.'))
  return [k for k in state_dict
          if k.endswith('.Conv_1.weight') or k.endswith('.NIN_3.W') or k == f'all_modules.{last}.weight']


def redraw_zero_init(state_dict, seed=1):
  """Copy of ``state_dict`` whose zero-initialised weights are re-drawn from the scale-1 variance-scaling init (fan_avg,
  uniform; layers.py:54-91), so that test outputs and activations are O(1) instead of ~1e-10 x."""
  g = torch.Generator().manual_seed(seed)
  out = dict(state_dict)
  for k in zero_init_keys(state_dict):
    w = state_dict[k]
    shape = tuple(w.shape)
    rf = np.prod(shape) / shape[0] / shape[1]
    fan_avg = (shape[0] * rf + shape[1] * rf) / 2     # symmetric in the two axes: NIN.W [in,out] and OIHW alike
    out[k] = ((torch.rand(*shape, generator=g, dtype=torch.float32) * 2. - 1.) * np.sqrt(3 / fan_avg)).to(w.device)
  return out
