"""The DDPM network (models/ddpm.py) without a GPU: the oracle against fixtures written by the real reference
(tools/make_golden_ddpm.py), the engine's parameter table against the module, parameter order, state_dict loading, the
registry and the options the engine does not implement."""
import json
import os

import pytest
import torch

from ddpm_helpers import golden_config, seeded_ddpm
from helpers import golden, rel_l2
from oracle import ddpm_oracle as DO
from oracle import sampling_oracle as SO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_oracle_matches_reference_forward_and_every_module_tiny():
  g = golden('ddpm_tiny.npz')
  cfg = golden_config('tiny')
  sd = seeded_ddpm(cfg).state_dict()
  taps = {}
  with torch.no_grad():
    y = DO.ddpm_forward(sd, cfg, torch.from_numpy(g['x']), torch.from_numpy(g['sigma']), taps=taps)
  assert sorted(taps) == sorted(int(k[3:]) for k in g if k.startswith('tap'))
  for i, v in taps.items():
    assert rel_l2(v, torch.from_numpy(g[f'tap{i}'])) < 1e-5, f'module {i}'
  assert rel_l2(y, torch.from_numpy(g['y'])) < 1e-5
  assert float(y.abs().mean()) > 0.1     # the re-drawn zero-init weights make the output O(1)


def test_oracle_matches_reference_forward_cifar10():
  g = golden('ddpm_cifar10.npz')
  cfg = golden_config('cifar10')
  sd = seeded_ddpm(cfg).state_dict()
  taps = {}
  with torch.no_grad():
    y = DO.ddpm_forward(sd, cfg, torch.from_numpy(g['x']), torch.from_numpy(g['sigma']), taps=taps)
  norms = torch.tensor([float(taps[i].double().norm()) for i in range(len(g['tap_norms']))], dtype=torch.float64)
  assert torch.allclose(norms, torch.from_numpy(g['tap_norms']), rtol=1e-4)
  assert rel_l2(y, torch.from_numpy(g['y'])) < 1e-4


@pytest.mark.parametrize('tag', ['vp_em_none', 'subvp_em_none', 'vp_ancestral_none'])
def test_oracle_sampler_matches_reference_tiny(tag):
  """The reference's get_pc_sampler at N=20 (continuous EM for VP / sub-VP, discrete-time ancestral sampling for VP)."""
  g = golden('pc_ddpm_tiny.npz')
  cfg = golden_config('tiny')
  sd = seeded_ddpm(cfg).state_dict()
  shape = g[tag].shape
  # (beta_max 10 for the ancestral run: at N=20, beta_max=20 makes the last discrete beta 1, see tools/make_golden_ddpm.py)
  sde = SO.SubVP(0.1, 20., 20) if tag.startswith('subvp') else SO.VP(0.1, 10. if 'ancestral' in tag else 20., 20)
  predictor = 'ancestral_sampling' if 'ancestral' in tag else 'euler_maruyama'
  torch.manual_seed({'vp_em_none': 41, 'subvp_em_none': 42, 'vp_ancestral_none': 43}[tag])
  with torch.no_grad():
    s, nfe = SO.pc_sample(sde, lambda a, l: DO.ddpm_forward(sd, cfg, a, l), shape, predictor, 'none', snr=0.16, n_steps=1,
                          eps=1e-3, continuous='ancestral' not in tag, denoise=True)
  assert nfe == int(g[tag + '_nfe'])
  assert rel_l2(s, torch.from_numpy(g[tag])) < 1e-4


@pytest.mark.parametrize('name,count', [('tiny', 685731), ('cifar10', 35218947), ('celebahq_256', 111569923)])
def test_engine_parameter_table_equals_module_parameters(name, count):
  model = seeded_ddpm(golden_config(name))
  table = model.native_param_table()
  assert table[0] == ('pos_freqs', (model.config.model.nf // 2,))     # the embedding's frequency table comes first
  assert [(n, tuple(p.shape)) for n, p in model.named_parameters()] == table[1:]
  assert sum(p.numel() for p in model.parameters()) == count


@pytest.mark.parametrize('name', ['tiny', 'cifar10'])
def test_parameter_order_matches_reference(name):
  ref = json.load(open(os.path.join(GOLDEN, 'ddpm_param_order.json')))[name]
  model = seeded_ddpm(golden_config(name))
  assert [[n, list(p.shape), bool(p.requires_grad)] for n, p in model.named_parameters()] == ref


def test_state_dict_keys_dtypes_and_strict_load_with_module_prefix():
  from score_sde_pytorch_b200.models.ddpm import DDPM
  cfg = golden_config('tiny')
  src = seeded_ddpm(cfg)
  sd = src.state_dict()
  assert sd['sigmas'].dtype == torch.float64 and 'pos_freqs' not in sd
  ref_keys = [e[0] for e in json.load(open(os.path.join(GOLDEN, 'ddpm_param_order.json')))['tiny']]
  assert [k for k in sd if k != 'sigmas'] == ref_keys
  for prefixed in (False, True):
    torch.manual_seed(9)
    dst = DDPM(cfg)
    v0 = dst._weights_version
    dst.load_state_dict({('module.' + k if prefixed else k): v for k, v in sd.items()}, strict=True)
    assert dst._weights_version > v0      # the packed engine copy is invalidated
    for k, v in dst.state_dict().items():
      assert torch.equal(v, sd[k]), k


def test_create_model_and_unsupported_options():
  from score_sde_pytorch_b200 import configs
  from score_sde_pytorch_b200.models import utils as mutils
  from score_sde_pytorch_b200.models.ddpm import DDPM
  for make in (configs.vp_cifar10_ddpm_continuous, configs.subvp_cifar10_ddpm_continuous, configs.vp_cifar10_ddpm,
               configs.tiny_ddpm):
    cfg = make()
    cfg.device = torch.device('cpu')
    assert type(mutils.create_model(cfg)) is DDPM
  assert configs.vp_cifar10_ddpm().training.continuous is False
  assert configs.vp_cifar10_ddpm().sampling.predictor == 'ancestral_sampling'
  for field, value in (('conditional', False), ('scale_by_sigma', True), ('resamp_with_conv', False),
                       ('nonlinearity', 'elu')):
    cfg = configs.tiny_ddpm()
    cfg.model[field] = value
    with pytest.raises(NotImplementedError):
      DDPM(cfg)


def test_engine_rejects_unsupported_family_configs():
  """b200_ncsnpp_create refuses DDPM without conditioning, with scale_by_sigma, and with GroupNorm channel counts that
  are not multiples of 32, with a message."""
  import ctypes
  from score_sde_pytorch_b200 import _lib
  model = seeded_ddpm(golden_config('tiny'))
  for field, value, text in (('conditional', 0, 'conditional'), ('scale_by_sigma', 1, 'scale_by_sigma'),
                             ('nf', 48, 'multiple of 32'), ('family', 2, 'family')):
    c = model._native_config()
    setattr(c, field, value)
    h = ctypes.c_void_p()
    with pytest.raises(RuntimeError, match=text):
      _lib.call('b200_ncsnpp_create', ctypes.byref(c), ctypes.byref(h))


def test_engine_plumbing_is_shared():
  """NCSNpp and DDPM use one engine base; the native samplers accept either."""
  from score_sde_pytorch_b200.models._engine import EngineModel
  from score_sde_pytorch_b200.models.ddpm import DDPM
  from score_sde_pytorch_b200.models.ncsnpp import NCSNpp
  assert issubclass(DDPM, EngineModel) and issubclass(NCSNpp, EngineModel)
  for attr in ('engine', 'forward', 'tap', 'load_state_dict', '_release', 'activation_range_report', 'invalidate_weights'):
    assert attr not in DDPM.__dict__ and attr not in NCSNpp.__dict__, attr
  model = seeded_ddpm(golden_config('tiny'))
  with pytest.raises(RuntimeError, match='CUDA'):
    model(torch.zeros(1, 3, 16, 16), torch.zeros(1))
