"""Golden fixtures for the DDPM++ family (configs/vp/cifar10_ddpmpp_continuous.py) from the REAL reference,
same recipe as tools/make_golden.py: this repository's deterministic weights are loaded into the reference's NCSNpp with
load_state_dict(strict=True) (fir=False naive resampling, positional embedding, no input pyramid), then

  ncsnpp_tiny_ddpmpp.npz      forward at batch 2 with every all_modules[i] activation (nf=32, 16x16)
  ncsnpp_cifar10_ddpmpp.npz   forward of the full-size CIFAR-10 DDPM++ (init_scale=1), output + per-module norms
  pc_ddpmpp_tiny.npz          the config's own sampler (VP SDE, EulerMaruyama + NoneCorrector, 20 steps), and the
                              sub-VP variant, through the reference's get_pc_sampler

    python tools/make_golden_ddpmpp.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
from score_sde_pytorch_b200 import configs as our_configs   # noqa: E402


def ddpmpp_configs():
  cifar = our_configs.vp_cifar10_ddpmpp_continuous()
  cifar.model.init_scale = 1.0
  return {'tiny_ddpmpp': (our_configs.tiny_ddpmpp(), 2), 'cifar10_ddpmpp': (cifar, 2)}


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, ncsnpp, mutils, _ = MG.import_reference()
  for name, (cfg, B) in ddpmpp_configs().items():
    cfg.device = torch.device('cpu')
    sd = MG.our_weights(cfg)
    torch.manual_seed(0)
    ref_model = mutils.get_model('ncsnpp')(cfg).eval()
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
    if name == 'tiny_ddpmpp':
      for i, v in taps.items():
        rec[f'tap{i}'] = v.numpy()
    else:
      rec['tap_norms'] = np.array([float(taps[i].double().norm()) if i in taps else 0.0
                                   for i in range(len(ref_model.all_modules))])
    np.savez_compressed(os.path.join(MG.OUT, f'ncsnpp_{name}.npz'), **rec)
    print(name, 'forward done', float(y.abs().mean()), 'modules', len(ref_model.all_modules))
    if name == 'tiny_ddpmpp':
      shape = (B, C, R, R)
      out = {}
      for tag, sde, seed in (('vp_em_none', sde_lib.VPSDE(beta_min=0.1, beta_max=20., N=20), 41),
                             ('subvp_em_none', sde_lib.subVPSDE(beta_min=0.1, beta_max=20., N=20), 42)):
        fn = sampling.get_pc_sampler(sde, shape, sampling.EulerMaruyamaPredictor, sampling.NoneCorrector, lambda v: v,
                                     snr=0.16, n_steps=1, probability_flow=False, continuous=True, denoise=True,
                                     eps=1e-3, device='cpu')
        torch.manual_seed(seed)
        s, nfe = fn(ref_model)
        out[tag] = s.numpy(); out[tag + '_nfe'] = nfe
      np.savez_compressed(os.path.join(MG.OUT, 'pc_ddpmpp_tiny.npz'), **out)
      print('pc written', {k: getattr(v, 'shape', v) for k, v in out.items()})


if __name__ == '__main__':
  main()
