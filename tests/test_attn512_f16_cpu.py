"""`precision='f16'` on the networks with 512-channel attention at 16x16 (T = 256, C = 512): the 256-pixel DDPM configs
and FFHQ-1024 NCSN++.  The engine plans them without a device; the fused core's C-ABI refuses C = 512 in TF32."""
import ctypes

import pytest

from score_sde_pytorch_b200 import _lib, configs
from score_sde_pytorch_b200.models.ddpm import DDPM
from score_sde_pytorch_b200.models.ncsnpp import NCSNpp

NETWORKS = {
    'celebahq_256_ddpm': (DDPM, configs.vp_celebahq_256_ddpm),
    'ffhq_1024_ncsnpp': (NCSNpp, configs.ve_ffhq_1024_ncsnpp_continuous),
}


@pytest.mark.parametrize('name', sorted(NETWORKS))
def test_f16_plans_networks_with_512_channel_attention(name):
  cls, cfg = NETWORKS[name]
  model = cls(cfg(), precision='f16')
  lib = _lib.load()
  h = ctypes.c_void_p()
  _lib.call('b200_ncsnpp_create', ctypes.byref(model._native_config()), ctypes.byref(h))
  try:
    for batch in (1, 8):
      ws = lib.b200_ncsnpp_workspace_bytes(h, batch)
      assert ws > 0, f'batch {batch}: {_lib.last_error()}'
  finally:
    lib.b200_ncsnpp_destroy(h)


def test_attention_core_refuses_c512_with_tf32_operands():
  lib = _lib.load()
  rc = lib.b200_attention_core_f32(None, None, None, None, None, None, None, None, 1, 256, 512, 1.0, 0, None)
  assert rc != 0
  err = _lib.last_error()
  assert 'C=512' in err and 'tf32' in err, err
