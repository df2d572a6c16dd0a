"""Golden fixtures for the probability-flow ODE sampler (sampling.py:414-485) from the REAL reference:
get_ode_sampler (scipy RK45, rtol = atol = 1e-5) on the reference's own NCSNpp with this repository's deterministic
weights, on CPU, for a fixed latent z.  ode_tiny.npz: per case z, samples, nfe.

    python tools/make_golden_ode.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
import make_golden_ddpmpp as MD   # noqa: E402


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, ncsnpp, mutils, _ = MG.import_reference()
  cfgs = dict(MG.golden_configs())
  cfgs.update(MD.ddpmpp_configs())
  out = {}
  cases = (('ve', 'tiny', lambda: sde_lib.VESDE(sigma_min=0.01, sigma_max=50, N=1000), 1e-5, False),
           ('vp', 'tiny_ddpmpp', lambda: sde_lib.VPSDE(beta_min=0.1, beta_max=20., N=1000), 1e-3, False),
           ('subvp', 'tiny_ddpmpp', lambda: sde_lib.subVPSDE(beta_min=0.1, beta_max=20., N=1000), 1e-3, True))
  for tag, name, mk, eps, denoise in cases:
    cfg, B = cfgs[name]
    cfg.device = torch.device('cpu')
    sd = MG.our_weights(cfg)
    torch.manual_seed(0)
    m = mutils.get_model('ncsnpp')(cfg).eval()
    m.load_state_dict(sd, strict=True)
    sde = mk()
    shape = (B, cfg.data.num_channels, cfg.data.image_size, cfg.data.image_size)
    torch.manual_seed(51)
    z = sde.prior_sampling(shape)
    fn = sampling.get_ode_sampler(sde, shape, lambda v: v, denoise=denoise, rtol=1e-5, atol=1e-5, method='RK45', eps=eps, device='cpu')
    torch.manual_seed(52)
    s, nfe = fn(m, z=z.clone())
    out[tag + '_z'] = z.numpy(); out[tag] = s.numpy(); out[tag + '_nfe'] = nfe
    print(tag, 'nfe', nfe, 'mean |x|', float(s.abs().mean()))
  np.savez_compressed(os.path.join(MG.OUT, 'ode_tiny.npz'), **out)


if __name__ == '__main__':
  main()
