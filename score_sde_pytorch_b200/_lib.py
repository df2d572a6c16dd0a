"""ctypes binding of ``libscoresde_b200.so`` (the C ABI in ``include/scoresde_b200.h``).

There is no CPU fallback: if the library is missing it is built with nvcc
(``build.py``); if that is impossible the import of anything that needs a device
kernel raises.  ``call(name, *args)`` turns a non-zero status into a
``RuntimeError`` carrying ``b200_last_error()`` — the analogue of the reference's
``TORCH_CHECK`` failures (``op/upfirdn2d.cpp:8,15-16``).
"""
import ctypes
import os
import threading

from . import build as _build

_LOCK = threading.Lock()
_LIB = None

c_void_p, c_int, c_ll, c_ull, c_float = (ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong,
                                         ctypes.c_ulonglong, ctypes.c_float)
c_char_p = ctypes.c_char_p
P = ctypes.POINTER


class NcsnppConfig(ctypes.Structure):
  """``b200_ncsnpp_config`` (include/scoresde_b200.h)."""
  _fields_ = [('image_size', c_int), ('num_channels', c_int), ('nf', c_int), ('num_res_blocks', c_int),
              ('num_levels', c_int), ('ch_mult', c_int * 8),
              ('num_attn_resolutions', c_int), ('attn_resolutions', c_int * 8),
              ('centered', c_int), ('scale_by_sigma', c_int), ('skip_rescale', c_int), ('conditional', c_int),
              ('progressive_input', c_int),
              ('fir_taps', c_int), ('fir_kernel', c_float * 8),
              ('precision', c_int), ('keep_activations', c_int), ('lanes', c_int),
              ('cuda_core_head', c_int), ('embedding_type', c_int), ('naive_resample', c_int), ('progressive', c_int), ('pdl', c_int),
              ('no_halo', c_int), ('family', c_int), ('tangent', c_int)]


class PcConfig(ctypes.Structure):
  """``b200_pc_config`` (include/scoresde_b200.h)."""
  _fields_ = [('n_steps', c_int), ('corrector', c_int), ('predictor', c_int), ('n_corrector_steps', c_int),
              ('snr', c_float),
              ('label', P(c_float)), ('score_scale', P(c_float)), ('alpha', P(c_float)),
              ('pa', P(c_float)), ('pb', P(c_float)), ('pc', P(c_float)),
              ('ca', P(c_float)), ('cb', P(c_float)), ('cc', P(c_float)),
              ('constraint', c_int), ('cm', P(c_float)), ('cs', P(c_float)),
              ('color_m', c_float * 9), ('color_minv', c_float * 9), ('noise_nhwc', c_int)]


# name -> (restype, argtypes); must list every symbol declared in include/scoresde_b200.h
SIGNATURES = {
  'b200_last_error': (c_char_p, []),
  'b200_version': (c_int, []),
  'b200_device_sm_count': (c_int, [P(c_int)]),
  'b200_upfirdn2d_f32': (c_int, [c_void_p, P(c_float), c_void_p] + [c_int] * 14 + [c_void_p]),
  'b200_fused_bias_act_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int,
                                      c_float, c_float, c_void_p]),
  'b200_groupnorm_nhwc_f32': (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                      c_float, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
  'b200_softmax_rows_f32': (c_int, [c_void_p, c_void_p, c_ll, c_int, c_float, c_int, c_void_p]),
  'b200_randn_like_torch_f32': (c_int, [c_void_p, c_ll, c_ull, c_ull, P(c_ull), c_void_p, c_void_p]),
  'b200_conv_nhwc_f32': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                 c_int, c_void_p, c_ll, c_void_p, c_float, c_int, c_void_p, c_int, c_void_p]),
  'b200_conv_skip_nhwc_f32': (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_float, c_int, c_void_p, c_void_p]),
  'b200_attention_core_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int, c_int, c_int, c_float, c_int, c_void_p]),
  'b200_attention_flash_f16': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
  'b200_conv_dilated_nhwc_f32': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                         c_int, c_void_p, c_int, c_void_p]),
  'b200_instnorm_plus_nhwc_f32': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                          c_void_p, c_void_p]),
  'b200_maxpool5_nhwc_f32': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
  'b200_bilinear_add_nhwc_f32': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
  'b200_pack_conv_weight_f32': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
  'b200_gemm_nt_f32': (c_int, [c_void_p, c_ll, c_int, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, c_void_p,
                               c_int, c_void_p, c_ll, c_int, c_void_p]),
  'b200_ncsnpp_create': (c_int, [P(NcsnppConfig), P(c_void_p)]),
  'b200_ncsnpp_destroy': (None, [c_void_p]),
  'b200_ncsnpp_num_params': (c_int, [c_void_p]),
  'b200_ncsnpp_param_info': (c_int, [c_void_p, c_int, c_char_p, c_int, P(c_ll), P(c_int)]),
  'b200_ncsnpp_weights_bytes': (c_ll, [c_void_p]),
  'b200_ncsnpp_bind_weights': (c_int, [c_void_p, c_void_p]),
  'b200_ncsnpp_load_param': (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
  'b200_ncsnpp_num_ops': (c_ll, [c_void_p]),
  'b200_ncsnpp_op_info': (c_int, [c_void_p, c_ll, c_char_p, c_int, P(c_int), P(ctypes.c_double)]),
  'b200_ncsnpp_op_bytes': (c_int, [c_void_p, c_ll, P(ctypes.c_double)]),
  'b200_ncsnpp_profile_ops': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_ll]),
  'b200_ncsnpp_workspace_bytes': (c_ll, [c_void_p, c_int]),
  'b200_ncsnpp_bind_workspace': (c_int, [c_void_p, c_int, c_void_p, c_ll]),
  'b200_ncsnpp_forward': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
  'b200_ncsnpp_tap': (c_int, [c_void_p, c_int, c_void_p, c_ll, P(c_int), c_void_p]),
  'b200_ncsnpp_launches_per_forward': (c_ll, [c_void_p]),
  'b200_ncsnpp_jvp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
  'b200_ncsnpp_tap_tangent': (c_int, [c_void_p, c_int, c_void_p, c_ll, P(c_int), c_void_p]),
  'b200_ncsnpp_profile_forward': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                          P(c_float), P(ctypes.c_double), P(c_ll)]),
  'b200_pc_create': (c_int, [c_void_p, P(PcConfig), c_int, P(c_void_p)]),
  'b200_pc_destroy': (None, [c_void_p]),
  'b200_pc_workspace_bytes': (c_ll, [c_void_p]),
  'b200_pc_bind_workspace': (c_int, [c_void_p, c_void_p, c_ll, c_void_p]),
  'b200_pc_run': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_ull, c_ull, P(c_ull), c_int, c_void_p]),
  'b200_pc_bind_constraint': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
  'b200_pc_step_external': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
  'b200_pc_launches_per_step': (c_ll, [c_void_p]),
  'b200_ode_stage_f64': (c_int, [c_void_p, c_void_p, c_ll, P(ctypes.c_double), c_int, ctypes.c_double, c_void_p, c_void_p, c_void_p]),
  'b200_ode_drift_f64': (c_int, [c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_void_p]),
  'b200_ode_div_f64': (c_int, [c_void_p, c_void_p, c_int, c_ll, c_void_p, c_void_p, c_void_p]),
  'b200_ode_workspace_doubles': (c_ll, []),
  'b200_ode_error_sumsq_f64': (c_int, [c_void_p, c_void_p, c_void_p, c_ll, P(ctypes.c_double), c_int, ctypes.c_double,
                                       ctypes.c_double, ctypes.c_double, c_void_p, c_void_p]),
  'b200_ode_error_sumsq2_f64': (c_int, [c_void_p, c_void_p, c_void_p, c_ll, P(ctypes.c_double), P(ctypes.c_double), c_int,
                                        ctypes.c_double, ctypes.c_double, c_void_p, c_void_p]),
  'b200_ode_scaled_sumsq_f64': (c_int, [c_void_p, c_void_p, c_void_p, c_ll, ctypes.c_double, ctypes.c_double, c_void_p, c_void_p]),
  'b200_dsm_perturb_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_ll, c_void_p]),
  'b200_dsm_workspace_doubles': (c_ll, [c_int, c_ll]),
  'b200_dsm_loss_f32': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_ll, c_int, c_int, c_void_p, c_void_p]),
}


def library_path():
  return _build.LIB


def load():
  """Load (building first if necessary) the native library.  Raises on failure."""
  global _LIB
  with _LOCK:
    if _LIB is not None:
      return _LIB
    # build() is a no-op when the in-tree .so matches the source digest; a stale or missing
    # library is rebuilt with nvcc (raises if that is impossible: there is no other code path)
    path = _build.build()
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
      fn = getattr(lib, name)   # AttributeError here == header/library mismatch; let it surface
      fn.restype = res
      fn.argtypes = args
    _LIB = lib
    return lib


def last_error():
  return load().b200_last_error().decode('utf-8', 'replace')


def call(name, *args):
  """Invoke an int-status entry point; raise ``RuntimeError`` with the library's message on failure."""
  lib = load()
  rc = getattr(lib, name)(*args)
  if rc != 0:
    raise RuntimeError(f'{name} failed ({rc}): {lib.b200_last_error().decode("utf-8", "replace")}')
  return rc


def ptr(t):
  """Device (or host) pointer of a torch tensor as a ctypes void*; ``None`` -> NULL."""
  return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr(device=None):
  import torch
  return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
