"""Golden fixture of the likelihood computation (bits/dim) from the REAL reference, same recipe as
tools/make_golden_ddpm.py: this repository's deterministic weights are loaded with load_state_dict(strict=True) into the
reference's own networks, then the reference's ``likelihood.get_likelihood_fn`` runs on CPU.

  likelihood_tiny.npz   for net in (tiny_ddpm, tiny_ddpmpp), sde in (vp, subvp), hutchinson in (rademacher, gaussian):
                          {net}_{sde}_{hutchinson}_{bpd,z,nfe,eps}   the reference's (bpd, z, nfe) and the Hutchinson draw it
                                                                     made (torch.manual_seed(SEED) right before the call)
                        {net}_data        fixed data: uniformly dequantised 8-bit values in [0, 1], then the config's scaler
                        {net}_jvp_{x,labels,v,y,jv}   one (x, labels, v, net(x), J_net(x) v) tuple (autograd JVP)

    python tools/make_golden_likelihood.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
from score_sde_pytorch_b200 import configs as our_configs   # noqa: E402
from score_sde_pytorch_b200.models.ddpm import DDPM as OurDDPM   # noqa: E402
from score_sde_pytorch_b200.models.ncsnpp import NCSNpp as OurNCSNpp   # noqa: E402
from oracle import ddpm_oracle   # noqa: E402

SEED = 11
BATCH = 2


def likelihood_configs():
  """name -> (config, reference model name); tests/test_likelihood_cpu.py builds the same."""
  return {'tiny_ddpm': (our_configs.tiny_ddpm(), 'ddpm'), 'tiny_ddpmpp': (our_configs.tiny_ddpmpp(), 'ncsnpp')}


def our_weights(name, cfg):
  torch.manual_seed(0)
  if name == 'tiny_ddpm':
    return ddpm_oracle.redraw_zero_init(OurDDPM(cfg).state_dict())
  return OurNCSNpp(cfg).state_dict()


def fixed_data(cfg, seed=3):
  g = torch.Generator().manual_seed(seed)
  R, C = cfg.data.image_size, cfg.data.num_channels
  x = (torch.randint(0, 256, (BATCH, C, R, R), generator=g).float() + torch.rand(BATCH, C, R, R, generator=g)) / 256.
  return x * 2. - 1. if cfg.data.centered else x     # datasets.get_data_scaler


def main():
  torch.set_num_threads(8)
  sde_lib, _, _, mutils, _ = MG.import_reference()
  from models import ddpm as _ref_ddpm   # noqa: F401  (registers 'ddpm')
  import likelihood as ref_likelihood
  out = {}
  for name, (cfg, ref_name) in likelihood_configs().items():
    cfg.device = torch.device('cpu')
    torch.manual_seed(0)
    model = mutils.get_model(ref_name)(cfg).eval()
    model.load_state_dict(our_weights(name, cfg), strict=True)
    data = fixed_data(cfg)
    out[f'{name}_data'] = data.numpy()
    inverse_scaler = (lambda x: (x + 1.) / 2.) if cfg.data.centered else (lambda x: x)
    for sde_name, sde in (('vp', sde_lib.VPSDE(beta_min=0.1, beta_max=20., N=1000)),
                          ('subvp', sde_lib.subVPSDE(beta_min=0.1, beta_max=20., N=1000))):
      for hutch in ('Rademacher', 'Gaussian'):
        fn = ref_likelihood.get_likelihood_fn(sde, inverse_scaler, hutchinson_type=hutch)
        torch.manual_seed(SEED)
        bpd, z, nfe = fn(model, data)
        torch.manual_seed(SEED)
        eps = torch.randn_like(data) if hutch == 'Gaussian' else torch.randint_like(data, low=0, high=2).float() * 2 - 1.
        key = f'{name}_{sde_name}_{hutch.lower()}'
        out[key + '_bpd'], out[key + '_z'], out[key + '_nfe'], out[key + '_eps'] = bpd.numpy(), z.numpy(), np.int64(nfe), eps.numpy()
        print(key, 'bpd', bpd.numpy(), 'nfe', nfe, flush=True)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(BATCH, cfg.data.num_channels, cfg.data.image_size, cfg.data.image_size, generator=g)
    v = torch.randn(x.shape, generator=g)
    labels = torch.tensor([731.3, 12.6])
    # torch.autograd.functional.jvp (the double-VJP form): forward-mode AD (torch.func.jvp) stops at the reference
    # AttnBlock's GroupNorm over a non-contiguous tensor
    y, jv = torch.autograd.functional.jvp(lambda xx: model(xx, labels), (x,), (v,))
    y, jv = y.detach(), jv.detach()
    for k, a in (('x', x), ('labels', labels), ('v', v), ('y', y), ('jv', jv)):
      out[f'{name}_jvp_{k}'] = a.numpy()
  path = os.path.join(MG.OUT, 'likelihood_tiny.npz')
  np.savez_compressed(path, **out)
  print('wrote', path)


if __name__ == '__main__':
  main()
