"""Golden fixtures for the NCSNv2 family (models/ncsnv2.py; configs/ve/ncsnv2/*.py) from the reference, same recipe as
tools/make_golden_ddpm.py: this repository's deterministic weights (``NCSNv2(config)`` under ``torch.manual_seed(0)``;
``ncsn_conv3x3`` keeps PyTorch's default initialisation, so nothing is re-drawn) are loaded into the reference's network
with load_state_dict(strict=True), then

  ncsnv2_tiny.npz          forward at batch 2 with every block output (tap0 begin_conv, then the ResidualBlocks, then the
                           RefineBlocks; nf=32, 16x16, 20 noise levels)
  ncsnv2_cifar10.npz       forward of the full-size CIFAR-10 NCSNv2, output + per-block norms
  ncsnv2_param_order.json  the reference networks' parameter lists (name, shape, requires_grad) in parameters() order, for
                           the tiny, CIFAR-10, CelebA and bedroom configurations
  pc_ncsnv2_tiny.npz       the reference's get_pc_sampler with NonePredictor + AnnealedLangevinDynamics, N = 20,
                           continuous=False, on the tiny network

The reference's NCSNv2 does not run as shipped, for three reasons the tool works around at run time without touching
the reference tree:
  * ``ncsn_conv3x3`` (layers.py:108-115) scales ``conv.bias`` even for ``bias=False`` (every RCU and CRP convolution),
    which raises AttributeError;
  * it pads every 3x3 convolution by 1 whatever its dilation, so the dilated ResidualBlocks shrink their input and the
    shortcut no longer matches (RuntimeError in res3).  The tool's replacement pads by the dilation, as the NCSNv2
    paper's network does;
  * the constructor reads ``config.data.channels``, which the default configs do not define
    (``configs.ve_cifar10_ncsnv2()`` sets it).
The sampler fixture meets a fourth: ``output / used_sigmas`` is float64 (the ``sigmas`` buffer is), so the ALD loop's
state becomes float64 after the first step, which the network's fp32 convolutions then reject.  The sampler runs the
reference network behind a wrapper that casts its input to float32 - what the engine's forward does - and keeps the
float64 output and state.

    python tools/make_golden_ncsnv2.py
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
from score_sde_pytorch_b200 import configs as our_configs   # noqa: E402
from score_sde_pytorch_b200.models import ncsnv2 as our_ncsnv2   # noqa: E402


def ncsnv2_configs():
  """name -> (config, batch); tests/ncsnv2_helpers.py:golden_config builds the same."""
  return {'tiny': (our_configs.tiny_ncsnv2(), 2), 'cifar10': (our_configs.ve_cifar10_ncsnv2(), 2),
          'celeba': (our_configs.ve_celeba_ncsnv2(), None), 'bedroom': (our_configs.ve_bedroom_ncsnv2(), None)}


def our_weights(cfg, seed=0):
  torch.manual_seed(seed)
  cls = our_ncsnv2.NCSNv2_128 if cfg.model.name == 'ncsnv2_128' else our_ncsnv2.NCSNv2
  return cls(cfg).state_dict()


def _conv3x3(in_planes, out_planes, stride=1, bias=True, dilation=1, init_scale=1., padding=None):
  """``ncsn_conv3x3`` with an optional bias and padding = dilation by default (see the module docstring)."""
  init_scale = 1e-10 if init_scale == 0 else init_scale
  conv = nn.Conv2d(in_planes, out_planes, stride=stride, bias=bias, dilation=dilation,
                   padding=dilation if padding is None else padding, kernel_size=3)
  conv.weight.data *= init_scale
  if conv.bias is not None:
    conv.bias.data *= init_scale
  return conv


class _Fp32Input(nn.Module):
  """The reference network with its input cast to float32 (its output stays float64)."""

  def __init__(self, net):
    super().__init__()
    self.net = net

  def forward(self, x, y):
    return self.net(x.float(), y)


def block_outputs(ref_model):
  """Forward hooks recording the engine's tap order: begin_conv, res*.*, refine*."""
  mods = [ref_model.begin_conv]
  L = 5 if hasattr(ref_model, 'res5') else 4
  for l in range(1, L + 1):
    mods += list(getattr(ref_model, f'res{l}'))
  mods += [getattr(ref_model, f'refine{k}') for k in range(1, L + 1)]
  return mods


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, _, mutils, _ = MG.import_reference()
  from models import layers, ncsnv2 as ref_ncsnv2   # noqa: F401  (registers 'ncsnv2_64' / 'ncsnv2_128')
  layers.ncsn_conv3x3 = _conv3x3
  order = {}
  for name, (cfg, B) in ncsnv2_configs().items():
    cfg.device = torch.device('cpu')
    sd = our_weights(cfg)
    torch.manual_seed(0)
    ref_model = mutils.get_model(cfg.model.name)(cfg).eval()
    order[name] = [[n, list(p.shape), bool(p.requires_grad)] for n, p in ref_model.named_parameters()]
    ref_model.load_state_dict(sd, strict=True)
    print(name, 'parameters', sum(p.numel() for p in ref_model.parameters()))
    if B is None:
      continue
    g = torch.Generator().manual_seed(7)
    R, C = cfg.data.image_size, cfg.data.num_channels
    x = torch.rand(B, C, R, R, generator=g)
    y = torch.tensor([3, cfg.model.num_scales - 2])[:B]
    mods = block_outputs(ref_model)
    taps, hooks = {}, []
    for i, mod in enumerate(mods):
      hooks.append(mod.register_forward_hook(lambda m, a, o, i=i: taps.__setitem__(i, o.detach().clone())))
    with torch.no_grad():
      out = ref_model(x, y)
    for h in hooks:
      h.remove()
    rec = dict(x=x.numpy(), y=y.numpy(), out=out.numpy())
    if name == 'tiny':
      for i, v in taps.items():
        rec[f'tap{i}'] = v.numpy()
    else:
      rec['tap_norms'] = np.array([float(taps[i].double().norm()) for i in range(len(mods))])
    np.savez_compressed(os.path.join(MG.OUT, f'ncsnv2_{name}.npz'), **rec)
    print(name, 'forward done', out.dtype, float(out.abs().mean()))
    if name == 'tiny':
      sde = sde_lib.VESDE(sigma_min=cfg.model.sigma_min, sigma_max=cfg.model.sigma_max, N=20)
      fn = sampling.get_pc_sampler(sde, (B, C, R, R), sampling.NonePredictor, sampling.AnnealedLangevinDynamics,
                                   lambda v: v, snr=cfg.sampling.snr, n_steps=2, probability_flow=False, continuous=False,
                                   denoise=True, eps=1e-5, device='cpu')
      torch.manual_seed(44)
      s, nfe = fn(_Fp32Input(ref_model))
      np.savez_compressed(os.path.join(MG.OUT, 'pc_ncsnv2_tiny.npz'), ald=s.numpy(), ald_nfe=nfe, ald_dtype=str(s.dtype))
      print('pc written', s.shape, s.dtype, nfe)
  path = os.path.join(MG.OUT, 'ncsnv2_param_order.json')
  json.dump(order, open(path, 'w'))
  print('wrote', path, {k: len(v) for k, v in order.items()})


if __name__ == '__main__':
  main()
