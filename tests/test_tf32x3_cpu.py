"""precision='tf32x3' (split TF32) without a GPU: the option reaches the engine, the parameter table is that of 'tf32', the
weight blob holds the extra lo copies, and the tangent pass accepts and refuses the same networks as in 'tf32'."""
import ctypes

import pytest

from ddpm_helpers import golden_config as ddpm_config, seeded_ddpm
from helpers import golden_config, seeded_model
from score_sde_pytorch_b200 import _lib, configs

NETS = {
    'cifar10_ve': lambda **kw: seeded_model(golden_config('cifar10_ve'), **kw),
    'cifar10_ddpmpp': lambda **kw: seeded_model(golden_config('cifar10_ddpmpp'), **kw),
    'cifar10_ddpm': lambda **kw: seeded_ddpm(ddpm_config('cifar10'), **kw),
    'tiny_progressive': lambda **kw: seeded_model(golden_config('tiny_progressive'), **kw),
}


def weights_bytes(model):
  cfg = model._native_config()
  h = ctypes.c_void_p()
  _lib.call('b200_ncsnpp_create', ctypes.byref(cfg), ctypes.byref(h))
  try:
    return _lib.load().b200_ncsnpp_weights_bytes(h)
  finally:
    _lib.load().b200_ncsnpp_destroy(h)


def test_precision_reaches_the_engine_config():
  model = NETS['cifar10_ddpmpp'](precision='tf32x3')
  assert model.precision == 'tf32x3' and model._native_config().precision == 3
  cfg = golden_config('cifar10_ddpmpp')
  cfg.model.precision = 'TF32x3'
  assert seeded_model(cfg)._native_config().precision == 3


@pytest.mark.parametrize('name', sorted(NETS))
def test_parameter_table_equals_tf32(name):
  assert NETS[name](precision='tf32x3').native_param_table() == NETS[name](precision='tf32').native_param_table()


@pytest.mark.parametrize('name', ['cifar10_ve', 'cifar10_ddpmpp', 'cifar10_ddpm'])
def test_weight_blob_holds_the_lo_copies(name):
  assert weights_bytes(NETS[name](precision='tf32x3')) > weights_bytes(NETS[name](precision='tf32'))

@pytest.mark.parametrize('name', ['cifar10_ddpm', 'cifar10_ddpmpp'])
def test_jvp_supported_for_ddpm_and_ddpmpp(name):
  NETS[name](precision='tf32x3').check_jvp_supported()


def test_jvp_still_refused_for_fir_resampling():
  model = seeded_model(configs.tiny_ncsnpp(), precision='tf32x3')
  with pytest.raises(NotImplementedError, match='naive_resample'):
    model.check_jvp_supported()


def test_unknown_precision_is_refused():
  with pytest.raises(ValueError):
    NETS['cifar10_ddpmpp'](precision='tf32x2')._native_config()
  cfg = NETS['cifar10_ddpmpp'](precision='tf32')._native_config()
  cfg.precision = 4
  h = ctypes.c_void_p()
  assert _lib.load().b200_ncsnpp_create(ctypes.byref(cfg), ctypes.byref(h)) != 0
  assert 'precision' in _lib.last_error()
