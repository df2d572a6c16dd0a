"""`precision='f16'` on attention shapes outside the fused core's T = 256: the flash fp16 core (attn_flash.cu) for T a
multiple of 128 up to 4096 and C = 128 / 256 / 512.  The engine plans the networks without a device; their tf32 plans
keep the sizes they had before the flash core existed; the new C-ABI entry point refuses what it does not implement."""
import ctypes

import pytest

from score_sde_pytorch_b200 import _lib, configs
from score_sde_pytorch_b200.models.ddpm import DDPM
from score_sde_pytorch_b200.models.ncsnpp import NCSNpp

# name -> (model class, config, attention (T, C) of the flash core,
#          tf32 (weight bytes, workspace bytes at batch 1, at batch 8) - the values of the planner without the flash core)
NETWORKS = {
    # DDPM++, nf = 64: 128 channels at 16x16
    'A_ddpmpp_T256_C128': (NCSNpp, lambda: configs.tiny_ddpmpp(nf=64, image_size=32, ch_mult=(1, 2, 2), attn_resolutions=(16,)),
                           (20377088, 2400256, 19173376)),
    # NCSN++ with attention at 32x32 (its 16x16 bottleneck keeps the fused T = 256, C = 256 core)
    'B_ncsnpp_T1024_C128': (NCSNpp, lambda: configs.tiny_ncsnpp(nf=64, image_size=32, ch_mult=(2, 4), attn_resolutions=(32,)),
                            (43035392, 7122944, 56963072)),
    # 64-pixel DDPM with attention at 32x32 (its 8x8 bottleneck keeps the small-token core)
    'C_ddpm_T1024_C128': (DDPM, lambda: configs.tiny_ddpm(nf=64, image_size=64, ch_mult=(1, 2, 2, 2), attn_resolutions=(32,)),
                          (24344320, 10564608, 84490240)),
    # attention at 64x64 (T = 4096, C = 128) and the 32x32 bottleneck (T = 1024, C = 256)
    'D_ddpm_T4096_C128': (DDPM, lambda: configs.tiny_ddpm(nf=128, image_size=64, ch_mult=(1, 2), attn_resolutions=(64,)),
                          (42560000, 79772672, 638162944)),
}


def _plan_sizes(model, batches=(1, 8)):
  lib = _lib.load()
  h = ctypes.c_void_p()
  _lib.call('b200_ncsnpp_create', ctypes.byref(model._native_config()), ctypes.byref(h))
  try:
    out = [lib.b200_ncsnpp_weights_bytes(h)]
    for batch in batches:
      ws = lib.b200_ncsnpp_workspace_bytes(h, batch)
      assert ws > 0, f'batch {batch}: {_lib.last_error()}'
      out.append(ws)
    return tuple(out)
  finally:
    lib.b200_ncsnpp_destroy(h)


@pytest.mark.parametrize('name', sorted(NETWORKS))
def test_f16_plans_networks_with_flash_attention_shapes(name):
  cls, cfg, _ = NETWORKS[name]
  _plan_sizes(cls(cfg(), precision='f16'))


@pytest.mark.parametrize('name', sorted(NETWORKS))
def test_tf32_plans_of_the_same_networks_are_unchanged(name):
  cls, cfg, tf32 = NETWORKS[name]
  assert _plan_sizes(cls(cfg(), precision='tf32')) == tf32


def test_attention_flash_entry_point_is_exported():
  lib = _lib.load()
  assert 'b200_attention_flash_f16' in _lib.SIGNATURES
  assert lib.b200_attention_flash_f16 is not None


@pytest.mark.parametrize('t,c', [(64, 128), (192, 128), (4224, 128), (8192, 128), (1024, 64), (1024, 384), (1024, 1024)])
def test_attention_flash_refuses_unsupported_shapes(t, c):
  lib = _lib.load()
  rc = lib.b200_attention_flash_f16(None, None, None, None, 1, t, c, None)
  assert rc != 0
  err = _lib.last_error()
  assert f'T={t} C={c}' in err, err


def test_attention_flash_refuses_null_pointers_and_empty_batches():
  lib = _lib.load()
  assert lib.b200_attention_flash_f16(None, None, None, None, 1, 1024, 128, None) != 0
  assert 'T=1024 C=128' in _lib.last_error()
  p = ctypes.c_void_p(16)   # never dereferenced: the argument check comes first
  assert lib.b200_attention_flash_f16(p, p, p, p, 0, 1024, 128, None) != 0
  err = _lib.last_error()
  assert 'nimg=0' in err and 'T=1024 C=128' in err, err


def test_attention_core_still_refuses_c512_with_tf32_operands():
  lib = _lib.load()
  rc = lib.b200_attention_core_f32(None, None, None, None, None, None, None, None, 1, 256, 512, 1.0, 0, None)
  assert rc != 0
  err = _lib.last_error()
  assert 'C=512' in err and 'tf32' in err, err
