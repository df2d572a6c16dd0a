"""``upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0))`` — FIR resampling on the sm_90a library.

Same call surface and result as the reference op (``op/upfirdn2d.py:145-156``): ``input`` is NCHW,
``kernel`` a 2-D FIR, ``up``/``down`` integer factors, ``pad=(pad0, pad1)`` applied to both axes.
The reference reshapes to ``[N*C, H, W, 1]`` before its pybind call (``op/upfirdn2d.py:99``) and so
does this wrapper; the engine itself calls the same kernel on NHWC with ``minor = C``.

Differentiable like the reference's ``UpFirDn2d`` / ``UpFirDn2dBackward`` pair (``op/upfirdn2d.py:19-141``): the
adjoint of an up/FIR/down pass is the same pass with the FIR flipped, ``up`` and ``down`` exchanged and the padding
``g_pad`` of ``:106-111``; the adjoint of that is the forward pass again (double backward, ``:66-85``).  All three run
on ``b200_upfirdn2d_f32``.  CPU tensors are rejected — the reference's pure-torch ``upfirdn2d_native`` fallback
(``:159-200``) is restated in ``oracle/``.
"""
import ctypes

import torch
from torch.autograd import Function

from .. import _lib


def _fir_pass(x, k, up, down, pad):
  """One native launch on ``[major, H, W, minor]`` (contiguous fp32 CUDA); ``up``/``down`` = (x, y), ``pad`` = (x0, x1, y0, y1)."""
  major, in_h, in_w, minor = x.shape
  kh, kw = k.shape
  out_h = (in_h * up[1] + pad[2] + pad[3] - kh) // down[1] + 1
  out_w = (in_w * up[0] + pad[0] + pad[1] - kw) // down[0] + 1
  y = torch.empty(major, out_h, out_w, minor, dtype=torch.float32, device=x.device)
  karr = (ctypes.c_float * (kh * kw))(*k.reshape(-1).tolist())
  with torch.cuda.device(x.device):
    _lib.call('b200_upfirdn2d_f32', _lib.ptr(x), karr, _lib.ptr(y), major, in_h, in_w, minor, kh, kw,
              up[0], up[1], down[0], down[1], pad[0], pad[1], pad[2], pad[3], _lib.stream_ptr(x.device))
  return y


def _host_fir(kernel):
  return kernel.detach().to('cpu', torch.float32).contiguous()


class UpFirDn2dBackward(Function):
  """grad_input of :class:`UpFirDn2d` as a differentiable op (``op/upfirdn2d.py:19-85``)."""

  @staticmethod
  def forward(ctx, grad_output, kernel, grad_kernel, up, down, pad, g_pad, in_size, out_size):
    g = grad_output.detach().to(torch.float32).reshape(-1, out_size[0], out_size[1], 1).contiguous()
    gi = _fir_pass(g, grad_kernel, down, up, g_pad)            # roles of up and down exchanged
    if tuple(gi.shape[1:3]) != (in_size[2], in_size[3]):
      raise RuntimeError(f'upfirdn2d backward: adjoint pass produced {tuple(gi.shape[1:3])}, input was {tuple(in_size[2:])}')
    ctx.kernel, ctx.up, ctx.down, ctx.pad, ctx.in_size, ctx.out_size = kernel, up, down, pad, in_size, out_size
    return gi.view(in_size)

  @staticmethod
  def backward(ctx, gradgrad_input):
    gg = gradgrad_input.detach().to(torch.float32).reshape(-1, ctx.in_size[2], ctx.in_size[3], 1).contiguous()
    out = _fir_pass(gg, ctx.kernel, ctx.up, ctx.down, ctx.pad)
    return out.view(ctx.in_size[0], ctx.in_size[1], ctx.out_size[0], ctx.out_size[1]), None, None, None, None, None, None, None, None


class UpFirDn2d(Function):
  """``UpFirDn2d.apply(input[N,C,H,W], kernel[kh,kw], (up_x, up_y), (down_x, down_y), (pad_x0, pad_x1, pad_y0, pad_y1))``
  (``op/upfirdn2d.py:88-141``)."""

  @staticmethod
  def forward(ctx, input, kernel, up, down, pad):
    if not input.is_cuda:
      raise RuntimeError('upfirdn2d (score_sde_pytorch_b200): input must be a CUDA tensor (no CPU path)')
    k = _host_fir(kernel)
    kh, kw = k.shape
    n, c, in_h, in_w = input.shape
    x = input.detach().to(torch.float32).reshape(n * c, in_h, in_w, 1).contiguous()
    out = _fir_pass(x, k, up, down, pad)
    out_h, out_w = out.shape[1], out.shape[2]
    ctx.kernel, ctx.grad_kernel = k, torch.flip(k, [0, 1]).contiguous()
    ctx.up, ctx.down, ctx.pad = tuple(up), tuple(down), tuple(pad)
    ctx.in_size, ctx.out_size = tuple(input.shape), (out_h, out_w)
    # padding of the adjoint pass (op/upfirdn2d.py:106-111)
    ctx.g_pad = (kw - pad[0] - 1, in_w * up[0] - out_w * down[0] + pad[0] - up[0] + 1,
                 kh - pad[2] - 1, in_h * up[1] - out_h * down[1] + pad[2] - up[1] + 1)
    return out.view(n, c, out_h, out_w)

  @staticmethod
  def backward(ctx, grad_output):
    gi = UpFirDn2dBackward.apply(grad_output, ctx.kernel, ctx.grad_kernel, ctx.up, ctx.down, ctx.pad, ctx.g_pad,
                                 ctx.in_size, ctx.out_size)
    return gi, None, None, None, None


def upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0)):
  if not input.is_cuda:
    raise RuntimeError('upfirdn2d (score_sde_pytorch_b200): input must be a CUDA tensor (no CPU path)')
  return UpFirDn2d.apply(input, kernel, (up, up), (down, down), (pad[0], pad[1], pad[0], pad[1]))


def upfirdn2d_nhwc(input, kernel, up=1, down=1, pad=(0, 0)):
  """Same op on a channels-last ``[N, H, W, C]`` tensor (the engine's internal layout); forward only."""
  x = input.detach().to(torch.float32).contiguous()
  return _fir_pass(x, _host_fir(kernel), (up, up), (down, down), (pad[0], pad[1], pad[0], pad[1]))
