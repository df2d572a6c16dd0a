"""ORACLE (test infrastructure, not product code): plain PyTorch fp32 restatement of the reference's NCSNv2 score
networks (``models/ncsnv2.py``: ``NCSNv2`` / ``'ncsnv2_64'`` and ``NCSNv2_128`` / ``'ncsnv2_128'``, with
``layers.py:133-310, 351-381, 453-507`` and ``normalization.py:157-183``).

Same rules as ``ncsnpp_oracle``: only tests, tools and benchmarks import it; ordinary torch ops in the reference's
operation order, NCHW.  Dilated 3x3 convolutions pad by their dilation, as the NCSNv2 paper's network does (the
reference's ``ncsn_conv3x3`` keeps padding 1, which makes the dilated blocks' shapes disagree; see
``tools/make_golden_ncsnv2.py``).  It is pinned against fixtures written by the reference (``tools/make_golden_ncsnv2.py``).
"""
import torch
import torch.nn.functional as F

# (output channels as multiples of nf, dilation) per level, and the RefineBlock widths; models/ncsnv2.py:60-100, 232-276
WALKS = {
  'ncsnv2_64': (((1, 1), (2, 1), (2, 2), (2, 4)), (2, 2, 1, 1)),
  'ncsnv2_128': (((1, 1), (2, 1), (2, 1), (4, 2), (4, 4)), (4, 2, 2, 1, 1)),
}


def in_plus(x, p, pre):
  """InstanceNorm2dPlus.forward (normalization.py:171-183)."""
  means = torch.mean(x, dim=(2, 3))
  m = torch.mean(means, dim=-1, keepdim=True)
  v = torch.var(means, dim=-1, keepdim=True)
  means = (means - m) / (torch.sqrt(v + 1e-5))
  h = F.instance_norm(x, eps=1e-5)
  h = h + means[..., None, None] * p[pre + '.alpha'][..., None, None]
  return p[pre + '.gamma'].view(1, -1, 1, 1) * h + p[pre + '.beta'].view(1, -1, 1, 1)


def _conv(x, p, pre, dilation=1):
  w = p[pre + '.weight']
  pad = dilation * (w.shape[-1] // 2)
  return F.conv2d(x, w, p.get(pre + '.bias'), padding=pad, dilation=dilation)


def _mean_pool(x):
  return sum([x[:, :, ::2, ::2], x[:, :, 1::2, ::2], x[:, :, ::2, 1::2], x[:, :, 1::2, 1::2]]) / 4.


def residual_block(x, p, pre, down, dilation):
  """ResidualBlock.forward (layers.py:494-507)."""
  h = F.elu(in_plus(x, p, pre + '.normalize1'))
  h = _conv(h, p, pre + '.conv1', dilation)
  h = F.elu(in_plus(h, p, pre + '.normalize2'))
  meanpool = down and dilation == 1
  if meanpool:   # ConvMeanPool (layers.py:365-369)
    h = _mean_pool(_conv(h, p, pre + '.conv2.conv'))
  else:
    h = _conv(h, p, pre + '.conv2', dilation)
  if meanpool:
    s = _mean_pool(_conv(x, p, pre + '.shortcut.conv'))
  elif (pre + '.shortcut.weight') in p:
    s = _conv(x, p, pre + '.shortcut', dilation)
  else:
    s = x
  return s + h


def rcu(x, p, pre, n_blocks):
  """RCUBlock.forward (layers.py:196-204)."""
  for i in range(n_blocks):
    residual = x
    for j in range(2):
      x = F.elu(x)
      x = _conv(x, p, f'{pre}.{i + 1}_{j + 1}_conv')
    x = x + residual
  return x


def refine_block(xs, p, pre, output_shape, end):
  """RefineBlock.forward (layers.py:296-310) with MSFBlock (:236-250) and CRPBlock(maxpool=True) (:133-154)."""
  hs = [rcu(x, p, f'{pre}.adapt_convs.{i}', 2) for i, x in enumerate(xs)]
  if len(xs) > 1:
    h = torch.zeros(xs[0].shape[0], p[f'{pre}.msf.convs.0.weight'].shape[0], *output_shape, device=xs[0].device)
    for i, hi in enumerate(hs):
      t = _conv(hi, p, f'{pre}.msf.convs.{i}')
      h = h + F.interpolate(t, size=output_shape, mode='bilinear', align_corners=True)
  else:
    h = hs[0]
  x = F.elu(h)
  path = x
  for i in range(2):
    path = F.max_pool2d(path, kernel_size=5, stride=1, padding=2)
    path = _conv(path, p, f'{pre}.crp.convs.{i}')
    x = path + x
  return rcu(x, p, f'{pre}.output_convs', 3 if end else 1)


def ncsnv2_forward(p, config, x, y, taps=None):
  """NCSNv2.forward / NCSNv2_128.forward (ncsnv2.py:107-132, 278-312) from a state dict ``p``.  ``y``: integer
  noise-level indices.  ``taps`` (optional dict) receives every block output under the engine's tap index: 0 begin_conv,
  then the ResidualBlocks, then the RefineBlocks."""
  levels, _ = WALKS[config.model.name]
  h = x if config.data.centered else 2 * x - 1.
  h = _conv(h, p, 'begin_conv')
  idx = 0
  if taps is not None:
    taps[idx] = h
  layers = []
  for lvl, (_, dil) in enumerate(levels):
    for b in range(2):
      h = residual_block(h, p, f'res{lvl + 1}.{b}', down=lvl > 0 and b == 0, dilation=dil)
      idx += 1
      if taps is not None:
        taps[idx] = h
    layers.append(h)
  L = len(levels)
  ref = None
  for k in range(1, L + 1):
    lay = layers[L - k]
    ref = refine_block([lay] if k == 1 else [lay, ref], p, f'refine{k}', lay.shape[2:], end=k == L)
    idx += 1
    if taps is not None:
      taps[idx] = ref
  out = _conv(F.elu(in_plus(ref, p, 'normalizer')), p, 'end_conv')
  used_sigmas = p['sigmas'][y].view(x.shape[0], *([1] * len(x.shape[1:])))
  return out / used_sigmas
