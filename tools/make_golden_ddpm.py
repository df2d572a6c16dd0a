"""Golden fixtures for the DDPM family (models/ddpm.py; configs/vp/ddpm/cifar10_continuous.py and friends) from the REAL
reference, same recipe as tools/make_golden_ddpmpp.py: this repository's deterministic weights (``DDPM(config)`` under
``torch.manual_seed(0)``, with the zero-initialised weights re-drawn at scale 1 by ``oracle.ddpm_oracle.redraw_zero_init``
so outputs and activations are not ~1e-10 x) are loaded into the reference's DDPM with load_state_dict(strict=True), then

  ddpm_tiny.npz           forward at batch 2 with every all_modules[i] activation (nf=32, ch_mult (1,2), 16x16)
  ddpm_cifar10.npz        forward of the full-size CIFAR-10 DDPM, output + per-module norms
  pc_ddpm_tiny.npz        the reference's get_pc_sampler at N=20 on the tiny network: VP and sub-VP Euler-Maruyama with no
                          corrector (continuous), and VP ancestral sampling with no corrector (continuous=False).  The
                          ancestral run uses beta_max=10: at N=20 the config's beta_max=20 makes the last discrete beta 1,
                          and the reference's ancestral update then divides by sqrt(1 - beta) = 0
  ddpm_param_order.json   the reference DDPM's parameter list (name, shape, requires_grad) in parameters() order

    python tools/make_golden_ddpm.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
from score_sde_pytorch_b200 import configs as our_configs   # noqa: E402
from score_sde_pytorch_b200.models.ddpm import DDPM as OurDDPM   # noqa: E402
from oracle import ddpm_oracle   # noqa: E402


def ddpm_configs():
  """name -> (config, batch); tests/ddpm_helpers.py:golden_config builds the same."""
  return {'tiny': (our_configs.tiny_ddpm(), 2), 'cifar10': (our_configs.vp_cifar10_ddpm_continuous(), 2)}


def our_weights(cfg, seed=0):
  torch.manual_seed(seed)
  return ddpm_oracle.redraw_zero_init(OurDDPM(cfg).state_dict())


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, _, mutils, _ = MG.import_reference()
  from models import ddpm as ref_ddpm   # noqa: F401  (registers 'ddpm')
  order = {}
  for name, (cfg, B) in ddpm_configs().items():
    cfg.device = torch.device('cpu')
    sd = our_weights(cfg)
    torch.manual_seed(0)
    ref_model = mutils.get_model('ddpm')(cfg).eval()
    order[name] = [[n, list(p.shape), bool(p.requires_grad)] for n, p in ref_model.named_parameters()]
    ref_model.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(7)
    R, C = cfg.data.image_size, cfg.data.num_channels
    x = torch.randn(B, C, R, R, generator=g) * 1.5
    labels = torch.linspace(999., 3., B) + 0.37          # VP labels t*999, deliberately non-integer
    with torch.no_grad():
      y = ref_model(x, labels)
      taps, hooks = {}, []
      for i, mod in enumerate(ref_model.all_modules):
        hooks.append(mod.register_forward_hook(lambda m, a, o, i=i: taps.__setitem__(i, o.detach().clone())))
      ref_model(x, labels)
      for h in hooks:
        h.remove()
    rec = dict(x=x.numpy(), sigma=labels.numpy(), y=y.numpy())
    if name == 'tiny':
      for i, v in taps.items():
        rec[f'tap{i}'] = v.numpy()
    else:
      rec['tap_norms'] = np.array([float(taps[i].double().norm()) if i in taps else 0.0
                                   for i in range(len(ref_model.all_modules))])
    np.savez_compressed(os.path.join(MG.OUT, f'ddpm_{name}.npz'), **rec)
    print(name, 'forward done', float(y.abs().mean()), 'modules', len(ref_model.all_modules),
          'parameters', sum(p.numel() for p in ref_model.parameters()))
    if name == 'tiny':
      shape = (B, C, R, R)
      out = {}
      for tag, sde, pred, continuous, seed in (
          ('vp_em_none', sde_lib.VPSDE(beta_min=0.1, beta_max=20., N=20), sampling.EulerMaruyamaPredictor, True, 41),
          ('subvp_em_none', sde_lib.subVPSDE(beta_min=0.1, beta_max=20., N=20), sampling.EulerMaruyamaPredictor, True, 42),
          ('vp_ancestral_none', sde_lib.VPSDE(beta_min=0.1, beta_max=10., N=20), sampling.AncestralSamplingPredictor, False, 43)):
        fn = sampling.get_pc_sampler(sde, shape, pred, sampling.NoneCorrector, lambda v: v, snr=0.16, n_steps=1,
                                     probability_flow=False, continuous=continuous, denoise=True, eps=1e-3, device='cpu')
        torch.manual_seed(seed)
        s, nfe = fn(ref_model)
        out[tag] = s.numpy(); out[tag + '_nfe'] = nfe
      np.savez_compressed(os.path.join(MG.OUT, 'pc_ddpm_tiny.npz'), **out)
      print('pc written', {k: getattr(v, 'shape', v) for k, v in out.items()})
  path = os.path.join(MG.OUT, 'ddpm_param_order.json')
  json.dump(order, open(path, 'w'))
  print('wrote', path, {k: len(v) for k, v in order.items()})


if __name__ == '__main__':
  main()
