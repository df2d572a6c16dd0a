"""Helpers of the DDPM tests: golden configs by name and the deterministic weights tools/make_golden_ddpm.py used."""
import torch

from score_sde_pytorch_b200 import configs
from oracle import ddpm_oracle


def golden_config(name):
  """Same constructions as tools/make_golden_ddpm.py:ddpm_configs() (plus the 256-pixel network, which has no golden)."""
  if name == 'tiny':
    return configs.tiny_ddpm()
  if name == 'cifar10':
    return configs.vp_cifar10_ddpm_continuous()
  if name == 'celebahq_256':
    return configs.vp_celebahq_256_ddpm()
  raise KeyError(name)


def seeded_ddpm(cfg, seed=0, **kw):
  """The engine-backed DDPM with the goldens' weights: constructed under ``torch.manual_seed(seed)``, then the weights the
  reference initialises at scale 0 re-drawn at scale 1 (oracle.ddpm_oracle.redraw_zero_init)."""
  from score_sde_pytorch_b200.models.ddpm import DDPM
  torch.manual_seed(seed)
  model = DDPM(cfg, **kw)
  model.load_state_dict(ddpm_oracle.redraw_zero_init(model.state_dict()))
  return model
