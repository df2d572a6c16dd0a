"""Golden fixture of the probability-flow ODE with scipy's other two explicit Runge-Kutta methods (RK23, DOP853) from the
REAL reference, same recipe as tools/make_golden_ode.py and tools/make_golden_likelihood.py: this repository's
deterministic weights are loaded with load_state_dict(strict=True) into the reference's own networks, then the
reference's ``sampling.get_ode_sampler`` and ``likelihood.get_likelihood_fn`` run on CPU with ``method=m``.

  ode_methods_tiny.npz   for m in (RK23, DOP853):
                           {m}_{case}, {m}_{case}_nfe         get_ode_sampler samples and nfe (rtol = atol = 1e-5) for
                                                              case in (ve: tiny NCSN++ / VE, vp_ddpm: tiny DDPM / VP,
                                                              vp_ddpmpp: tiny DDPM++ / VP)
                           {m}_lik_{net}_{bpd,z,nfe,eps}      get_likelihood_fn (VP, Rademacher, rtol = atol = 1e-5) for
                                                              net in (tiny_ddpm, tiny_ddpmpp), the Hutchinson draw it made
                                                              (torch.manual_seed(SEED) right before the call)
                         {case}_z        the sampler's latent (torch.manual_seed(51), sde.prior_sampling)
                         {net}_data      the likelihood's data (make_golden_likelihood.fixed_data)

    python tools/make_golden_ode_methods.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG   # noqa: E402
import make_golden_likelihood as ML   # noqa: E402

METHODS = ('RK23', 'DOP853')
SEED = 11


def main():
  torch.set_num_threads(8)
  sde_lib, sampling, _, mutils, _ = MG.import_reference()
  from models import ddpm as _ref_ddpm   # noqa: F401  (registers 'ddpm')
  import likelihood as ref_likelihood

  def reference_model(name):
    """(config, reference network with this repository's weights) for the fixture networks."""
    if name == 'tiny':
      cfg, _ = MG.golden_configs()['tiny']
      sd, ref_name = MG.our_weights(cfg), 'ncsnpp'
    else:
      cfg, ref_name = ML.likelihood_configs()[name]
      sd = ML.our_weights(name, cfg)
    cfg.device = torch.device('cpu')
    torch.manual_seed(0)
    model = mutils.get_model(ref_name)(cfg).eval()
    model.load_state_dict(sd, strict=True)
    return cfg, model

  out = {}
  vp = lambda: sde_lib.VPSDE(beta_min=0.1, beta_max=20., N=1000)
  for case, name, mk, eps in (('ve', 'tiny', lambda: sde_lib.VESDE(sigma_min=0.01, sigma_max=50, N=1000), 1e-5),
                              ('vp_ddpm', 'tiny_ddpm', vp, 1e-3),
                              ('vp_ddpmpp', 'tiny_ddpmpp', vp, 1e-3)):
    cfg, model = reference_model(name)
    sde = mk()
    shape = (ML.BATCH, cfg.data.num_channels, cfg.data.image_size, cfg.data.image_size)
    torch.manual_seed(51)
    z = sde.prior_sampling(shape)
    out[case + '_z'] = z.numpy()
    for m in METHODS:
      fn = sampling.get_ode_sampler(sde, shape, lambda v: v, rtol=1e-5, atol=1e-5, method=m, eps=eps, device='cpu')
      torch.manual_seed(52)
      s, nfe = fn(model, z=z.clone())
      out[f'{m}_{case}'], out[f'{m}_{case}_nfe'] = s.numpy(), np.int64(nfe)
      print(m, case, 'nfe', nfe, 'mean |x|', float(s.abs().mean()), flush=True)

  for name in ('tiny_ddpm', 'tiny_ddpmpp'):
    cfg, model = reference_model(name)
    data = ML.fixed_data(cfg)
    out[f'{name}_data'] = data.numpy()
    inverse_scaler = (lambda x: (x + 1.) / 2.) if cfg.data.centered else (lambda x: x)
    for m in METHODS:
      fn = ref_likelihood.get_likelihood_fn(vp(), inverse_scaler, hutchinson_type='Rademacher', method=m)
      torch.manual_seed(SEED)
      bpd, z, nfe = fn(model, data)
      torch.manual_seed(SEED)
      noise = torch.randint_like(data, low=0, high=2).float() * 2 - 1.
      key = f'{m}_lik_{name}'
      out[key + '_bpd'], out[key + '_z'], out[key + '_nfe'], out[key + '_eps'] = bpd.numpy(), z.numpy(), np.int64(nfe), noise.numpy()
      print(key, 'bpd', bpd.numpy(), 'nfe', nfe, flush=True)
  path = os.path.join(MG.OUT, 'ode_methods_tiny.npz')
  np.savez_compressed(path, **out)
  print('wrote', path)


if __name__ == '__main__':
  main()
