"""Helpers of the NCSNv2 tests: golden configs by name and the deterministic weights tools/make_golden_ncsnv2.py used."""
import torch

from score_sde_pytorch_b200 import configs


def golden_config(name):
  """Same constructions as tools/make_golden_ncsnv2.py:ncsnv2_configs()."""
  return {'tiny': configs.tiny_ncsnv2, 'cifar10': configs.ve_cifar10_ncsnv2, 'celeba': configs.ve_celeba_ncsnv2,
          'bedroom': configs.ve_bedroom_ncsnv2}[name]()


def seeded_ncsnv2(cfg, seed=0, **kw):
  """The engine-backed NCSNv2 with the goldens' weights: constructed under ``torch.manual_seed(seed)``."""
  from score_sde_pytorch_b200.models import ncsnv2
  torch.manual_seed(seed)
  cls = ncsnv2.NCSNv2_128 if cfg.model.name == 'ncsnv2_128' else ncsnv2.NCSNv2
  return cls(cfg, **kw)
