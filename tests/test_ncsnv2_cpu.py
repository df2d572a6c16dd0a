"""The NCSNv2 networks (models/ncsnv2.py) without a GPU: the oracle against fixtures written by the reference
(tools/make_golden_ncsnv2.py), the engine's parameter table against the module and the reference's parameter order,
state_dict loading, the registry, the options the engine refuses, and dry-run plans of the three shipped configurations."""
import ctypes
import json
import os

import pytest
import torch

from helpers import golden, rel_l2
from ncsnv2_helpers import golden_config, seeded_ncsnv2
from oracle import ncsnv2_oracle as VO
from oracle import sampling_oracle as SO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_oracle_matches_reference_forward_and_every_block_tiny():
  g = golden('ncsnv2_tiny.npz')
  cfg = golden_config('tiny')
  sd = seeded_ncsnv2(cfg).state_dict()
  taps = {}
  with torch.no_grad():
    out = VO.ncsnv2_forward(sd, cfg, torch.from_numpy(g['x']), torch.from_numpy(g['y']), taps=taps)
  assert sorted(taps) == sorted(int(k[3:]) for k in g if k.startswith('tap'))
  for i, v in taps.items():
    assert rel_l2(v, torch.from_numpy(g[f'tap{i}'])) < 1e-5, f'block {i}'
  assert out.dtype == torch.float64 and g['out'].dtype.name == 'float64'
  assert rel_l2(out, torch.from_numpy(g['out'])) < 1e-5


def test_oracle_matches_reference_forward_cifar10():
  g = golden('ncsnv2_cifar10.npz')
  cfg = golden_config('cifar10')
  sd = seeded_ncsnv2(cfg).state_dict()
  taps = {}
  with torch.no_grad():
    out = VO.ncsnv2_forward(sd, cfg, torch.from_numpy(g['x']), torch.from_numpy(g['y']), taps=taps)
  norms = torch.tensor([float(taps[i].double().norm()) for i in range(len(g['tap_norms']))], dtype=torch.float64)
  assert torch.allclose(norms, torch.from_numpy(g['tap_norms']), rtol=1e-5)
  assert rel_l2(out, torch.from_numpy(g['out'])) < 1e-5


def test_oracle_sampler_matches_reference_tiny():
  """The reference's get_pc_sampler at N=20 with NonePredictor + AnnealedLangevinDynamics (continuous=False)."""
  g = golden('pc_ncsnv2_tiny.npz')
  cfg = golden_config('tiny')
  sd = seeded_ncsnv2(cfg).state_dict()
  sde = SO.VE(cfg.model.sigma_min, cfg.model.sigma_max, 20)
  torch.manual_seed(44)
  with torch.no_grad():
    s, nfe = SO.pc_sample(sde, lambda a, l: VO.ncsnv2_forward(sd, cfg, a.float(), l), g['ald'].shape, 'none', 'ald',
                          snr=cfg.sampling.snr, n_steps=2, eps=1e-5, continuous=False, denoise=True)
  assert nfe == int(g['ald_nfe'])
  assert str(s.dtype) == str(g['ald_dtype'])
  assert rel_l2(s, torch.from_numpy(g['ald'])) < 1e-4


@pytest.mark.parametrize('name', ['tiny', 'cifar10', 'celeba', 'bedroom'])
def test_parameter_table_and_order_match_reference(name):
  ref = json.load(open(os.path.join(GOLDEN, 'ncsnv2_param_order.json')))[name]
  model = seeded_ncsnv2(golden_config(name))
  assert [[n, list(p.shape), bool(p.requires_grad)] for n, p in model.named_parameters()] == ref
  assert model.native_param_table() == [(n, tuple(p.shape)) for n, p in model.named_parameters()]
  assert sum(p.numel() for p in model.parameters()) == sum(int(torch.tensor(s).prod()) for _, s, _ in ref)


def test_state_dict_keys_dtypes_and_strict_load_with_module_prefix():
  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2
  cfg = golden_config('tiny')
  src = seeded_ncsnv2(cfg)
  sd = src.state_dict()
  assert sd['sigmas'].dtype == torch.float64 and sd['sigmas'].numel() == cfg.model.num_scales
  ref_keys = [e[0] for e in json.load(open(os.path.join(GOLDEN, 'ncsnv2_param_order.json')))['tiny']]
  assert [k for k in sd if k != 'sigmas'] == ref_keys
  for prefixed in (False, True):
    torch.manual_seed(9)
    dst = NCSNv2(cfg)
    v0 = dst._weights_version
    dst.load_state_dict({('module.' + k if prefixed else k): v for k, v in sd.items()}, strict=True)
    assert dst._weights_version > v0
    for k, v in dst.state_dict().items():
      assert torch.equal(v, sd[k]), k


def test_create_model_returns_the_new_classes():
  from score_sde_pytorch_b200 import configs
  from score_sde_pytorch_b200.models import utils as mutils
  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2, NCSNv2_128
  for make, cls in ((configs.ve_cifar10_ncsnv2, NCSNv2), (configs.ve_celeba_ncsnv2, NCSNv2),
                    (configs.ve_bedroom_ncsnv2, NCSNv2_128), (configs.tiny_ncsnv2, NCSNv2)):
    cfg = make()
    cfg.device = torch.device('cpu')
    assert type(mutils.create_model(cfg)) is cls
    assert cfg.training.continuous is False and cfg.sampling.predictor == 'none' and cfg.sampling.corrector == 'ald'


@pytest.mark.parametrize('field,value,text', [
    ('image_size', 28, 'image_size'), ('image_size', 96, 'image_size'), ('image_size', 30, 'image_size'),
    ('normalization', 'InstanceNorm', 'normalization'), ('normalization', 'GroupNorm', 'normalization'),
    ('nonlinearity', 'swish', 'nonlinearity'), ('interpolation', 'nearest', 'interpolation'),
    ('precision', 'tf32x3', 'precision')])
def test_unsupported_options_are_refused_with_the_field_name(field, value, text):
  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2
  cfg = golden_config('tiny')
  if field == 'image_size':
    cfg.data.image_size = value
  elif field == 'precision':
    cfg.model.precision = value
  else:
    cfg.model[field] = value
  with pytest.raises(NotImplementedError, match=text):
    NCSNv2(cfg)


def test_ncsnv2_128_refuses_sizes_outside_its_walk():
  from score_sde_pytorch_b200.models.ncsnv2 import NCSNv2_128
  cfg = golden_config('bedroom')
  cfg.data.image_size = 256
  with pytest.raises(NotImplementedError, match='image_size'):
    NCSNv2_128(cfg)


@pytest.mark.parametrize('name', ['ncsnv2_256', 'ncsn'])
def test_unimplemented_families_are_refused_by_name(name):
  from score_sde_pytorch_b200.models import utils as mutils
  cfg = golden_config('cifar10')
  cfg.model.name = name
  cfg.device = torch.device('cpu')
  with pytest.raises(NotImplementedError, match=name):
    mutils.create_model(cfg)


def test_tangent_pass_and_split_tf32_are_refused():
  """jvp / check_jvp_supported name the family; the engine refuses tangent = 1 and precision 3 for family 2 itself."""
  from score_sde_pytorch_b200 import _lib
  model = seeded_ncsnv2(golden_config('tiny'))
  with pytest.raises(NotImplementedError, match='NCSNv2'):
    model.check_jvp_supported()
  with pytest.raises(NotImplementedError, match='NCSNv2'):
    model.jvp(torch.zeros(1, 3, 16, 16), torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, 16, 16))
  for field, value in (('tangent', 1), ('precision', 3), ('num_levels', 3)):
    c = model._native_config()
    setattr(c, field, value)
    h = ctypes.c_void_p()
    with pytest.raises(RuntimeError, match='family = 2'):
      _lib.call('b200_ncsnpp_create', ctypes.byref(c), ctypes.byref(h))


def test_forward_refuses_continuous_labels_and_cpu_tensors():
  model = seeded_ncsnv2(golden_config('tiny'))
  with pytest.raises(TypeError, match='noise-level indices'):
    model(torch.zeros(1, 3, 16, 16), torch.ones(1))
  with pytest.raises(RuntimeError, match='CUDA'):
    model(torch.zeros(1, 3, 16, 16), torch.zeros(1, dtype=torch.long))


def _dry_plan(model, batch):
  from score_sde_pytorch_b200 import _lib
  lib = _lib.load()
  h = ctypes.c_void_p()
  cfg = model._native_config()
  _lib.call('b200_ncsnpp_create', ctypes.byref(cfg), ctypes.byref(h))
  try:
    return lib.b200_ncsnpp_weights_bytes(h), lib.b200_ncsnpp_workspace_bytes(h, batch)
  finally:
    lib.b200_ncsnpp_destroy(h)


@pytest.mark.parametrize('name', ['cifar10', 'celeba', 'bedroom'])
@pytest.mark.parametrize('precision', ['tf32', 'f16', 'fp32'])
def test_full_size_networks_plan(name, precision):
  """Weight and workspace bytes of a dry run at batch 1, 8 and 128: every block of the walk plans."""
  model = seeded_ncsnv2(golden_config(name), precision=precision)
  nparams = sum(p.numel() for p in model.parameters())
  prev = 0
  for batch in (1, 8, 128):
    wb, ws = _dry_plan(model, batch)
    assert wb >= 4 * nparams, (wb, nparams)
    assert ws > prev, (batch, ws)
    prev = ws
  R = model.config.data.image_size
  assert ws >= 128 * R * R * model.config.model.nf * 4   # at least one full-resolution activation of the batch


def test_tap_names_cover_every_block():
  m64 = seeded_ncsnv2(golden_config('tiny'))
  assert m64.tap_names() == ['begin_conv'] + [f'res{l}.{b}' for l in range(1, 5) for b in range(2)] + \
      [f'refine{k}' for k in range(1, 5)]
  m128 = seeded_ncsnv2(golden_config('bedroom'))
  assert len(m128.tap_names()) == 1 + 10 + 5
