"""Helpers for the `-m gpu` tests: thin ctypes callers of the C ABI on torch CUDA tensors and
the strict-fp32 GPU oracle setup."""
import ctypes

import torch

from score_sde_pytorch_b200 import _lib


def strict_fp32():
  """The oracle must not be blurred by TF32 (PyTorch lets cuDNN convs use it by default)."""
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.set_float32_matmul_precision('highest')


def round_tf32(x):
  """Round-to-nearest (ties away from zero, like cvt.rna.tf32.f32) onto the TF32 grid."""
  xi = x.contiguous().view(torch.int32)
  r = ((xi + 0x1000) & ~0x1FFF)
  return r.view(torch.float32)


def to_nhwc(x):
  return x.permute(0, 2, 3, 1).contiguous()


def to_nchw(x):
  return x.permute(0, 3, 1, 2).contiguous()


def pack_conv_weight(w, round_tf32_=False, f16=False):
  """OIHW fp32 -> [taps][O][I]; f16=True packs IEEE fp16 elements (operand mode 2)."""
  o, i, k, _ = w.shape
  out = torch.empty(k * k, o, i, device=w.device, dtype=torch.float16 if f16 else torch.float32)
  _lib.call('b200_pack_conv_weight_f32', _lib.ptr(w.contiguous()), _lib.ptr(out), o, i, k, 2 if f16 else int(round_tf32_),
            _lib.stream_ptr(w.device))
  return out


def conv_nhwc(x1, x2, wp, bias, cout, ksize, rowvec=None, rowvec_ld=0, residual=None, scale=1.0, round_out=False, impl=0):
  B, H, W, C1 = x1.shape
  C2 = x2.shape[3] if x2 is not None else 0
  out = torch.empty(B, H, W, cout, device=x1.device, dtype=torch.float32)
  _lib.call('b200_conv_nhwc_f32', _lib.ptr(x1), C1, _lib.ptr(x2), C2, B, H, W, _lib.ptr(wp), _lib.ptr(bias), cout,
            ksize, _lib.ptr(rowvec), rowvec_ld, _lib.ptr(residual), float(scale), int(round_out), _lib.ptr(out),
            impl, _lib.stream_ptr(x1.device))
  return out


def conv_skip_nhwc(x, s1, s2, wp, bias, wskip, bias_skip, cout, residual=None, scale=1.0, round_out=False):
  B, H, W, C = x.shape
  out = torch.empty(B, H, W, cout, device=x.device, dtype=torch.float32)
  _lib.call('b200_conv_skip_nhwc_f32', _lib.ptr(x), C, _lib.ptr(s1), s1.shape[3], _lib.ptr(s2),
            s2.shape[3] if s2 is not None else 0, B, H, W, _lib.ptr(wp), _lib.ptr(bias), _lib.ptr(wskip),
            _lib.ptr(bias_skip), cout, _lib.ptr(residual), float(scale), int(round_out), _lib.ptr(out),
            _lib.stream_ptr(x.device))
  return out


def attention_core(qk, vT, w3, bv, b3, x, out_scale, want_stats=False):
  """qk [nimg*T, 2C], vT [nimg, C, T], w3 [C, C] (out, in), x [nimg*T, C] -> out [nimg*T, C] (+ quad sums).
  fp16 qk/vT/w3 select the wgmma .f16 variant."""
  nimg, C, T = vT.shape
  f16 = qk.dtype == torch.float16
  assert vT.dtype == qk.dtype and w3.dtype == qk.dtype
  out = torch.empty_like(x)
  qs = torch.zeros(nimg, C // 4, 2, device=x.device, dtype=torch.float64) if want_stats else None
  _lib.call('b200_attention_core_f32', _lib.ptr(qk), _lib.ptr(vT), _lib.ptr(w3), _lib.ptr(bv), _lib.ptr(b3), _lib.ptr(x),
            _lib.ptr(out), _lib.ptr(qs), nimg, T, C, float(out_scale), int(f16), _lib.stream_ptr(x.device))
  return (out, qs) if want_stats else out


def gemm_nt(a, w, nbatch, m, n, k, lda=None, ldw=None, a_batch_rows=None, w_batch_rows=None, bias=None,
            round_out=False, impl=0):
  lda = k if lda is None else lda
  ldw = k if ldw is None else ldw
  a_batch_rows = m if a_batch_rows is None else a_batch_rows
  w_batch_rows = n if w_batch_rows is None else w_batch_rows
  out = torch.empty(nbatch * m, n, device=a.device, dtype=torch.float32)
  _lib.call('b200_gemm_nt_f32', _lib.ptr(a), lda, a_batch_rows, _lib.ptr(w), ldw, w_batch_rows, nbatch, m, n, k,
            _lib.ptr(bias), int(round_out), _lib.ptr(out), n, impl, _lib.stream_ptr(a.device))
  return out


_vp, _i, _ll, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float


class TcTestDesc(ctypes.Structure):
  """``b200_tc_test_desc`` (include/scoresde_b200.h); ``struct_bytes`` is filled in by ``tc_contract``."""
  _fields_ = [('struct_bytes', _i),
              ('a1', _vp), ('a2', _vp), ('c1', _i), ('c2', _i),
              ('conv', _i), ('h', _i), ('w', _i), ('nimg', _i), ('taps', _i), ('stride', _i), ('valid_pad', _i),
              ('hin', _i), ('win', _i), ('dilation', _i), ('no_halo', _i), ('f16', _i),
              ('a_rows', _ll), ('a_ld', _ll), ('a_batch_rows', _i),
              ('wt', _vp), ('n_total', _i), ('k_total', _i), ('w_rows', _ll), ('w_ld', _ll), ('w_batch_rows', _i),
              ('nbatch', _i), ('m_per_batch', _i),
              ('a3', _vp), ('a4', _vp), ('c3', _i), ('c4', _i), ('w2', _vp),
              ('split', _i), ('a1_lo', _vp), ('a2_lo', _vp), ('a3_lo', _vp), ('a4_lo', _vp), ('w_lo', _vp), ('w2_lo', _vp),
              ('qstats', _vp),
              ('bias', _vp), ('rowvec', _vp), ('rowvec_ld', _ll), ('residual', _vp), ('ld_res', _ll),
              ('per_img_div', _vp), ('div_stride', _ll), ('scale', _f), ('store_mode', _i), ('rows_per_img', _i),
              ('out', _vp), ('ld_out', _ll), ('out_nchw', _i), ('n_valid', _i)]


def tc_contract(device, struct_bytes=None, **fields):
  """One tensor-core contraction through ``b200_tc_contract_f32``.  Tensor-valued fields are passed as device pointers,
  the rest as given; returns the plan's form ("swap-halo", "single256", ...)."""
  d = TcTestDesc()
  d.struct_bytes = ctypes.sizeof(TcTestDesc) if struct_bytes is None else struct_bytes
  d.scale = 1.0
  for k, v in fields.items():
    setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
  form = ctypes.create_string_buffer(64)
  _lib.call('b200_tc_contract_f32', ctypes.byref(d), form, len(form),
            _lib.stream_ptr(device) if device is not None else None)
  return form.value.decode()


def randn_like_torch(numel, seed, offset, device):
  out = torch.empty(numel, device=device, dtype=torch.float32)
  ws = torch.zeros(2, device=device, dtype=torch.int64)
  inc = ctypes.c_ulonglong(0)
  _lib.call('b200_randn_like_torch_f32', _lib.ptr(out), numel, ctypes.c_ulonglong(seed), ctypes.c_ulonglong(offset),
            ctypes.byref(inc), _lib.ptr(ws), _lib.stream_ptr(device))
  return out, inc.value
