"""``fused_leaky_relu`` / ``FusedLeakyReLU`` on the sm_90a library.

Mirror of ``op/fused_act.py:20-97``: ``y = leaky_relu(x + bias[c], negative_slope) * scale`` with the bias broadcast over
dim 1, differentiable to second order like the reference's ``FusedLeakyReLUFunction`` / ``...Backward`` pair: the first
derivative is the same kernel gated on the saved OUTPUT (``fused_bias_act(grad, empty, out, 3, 1, ...)``, ``:27-29``), the
bias gradient its sum over every dim but 1 (``:31-36``), and the derivative of that is the gated kernel again (``:41-46``).
(No model in the reference calls it — it is compiled at import, ``op/__init__.py:1`` — but it is part of the native
surface, so it is kept.)
"""
import torch
from torch import nn
from torch.autograd import Function

from .. import _lib


def _bias_act(x, bias, ref, act, grad, negative_slope, scale):
  """``b200_fused_bias_act_f32`` on a contiguous fp32 CUDA tensor (bias over dim 1; ``ref`` gates when ``grad == 1``)."""
  x = x.detach().to(torch.float32).contiguous()
  b = None if bias is None or bias.numel() == 0 else bias.detach().to(device=x.device, dtype=torch.float32).contiguous()
  r = None if ref is None else ref.detach().to(torch.float32).contiguous()
  y = torch.empty_like(x)
  step_b = 1
  for d in x.shape[2:]:
    step_b *= d
  with torch.cuda.device(x.device):
    _lib.call('b200_fused_bias_act_f32', _lib.ptr(x), _lib.ptr(b), _lib.ptr(r), _lib.ptr(y), x.numel(), step_b,
              b.numel() if b is not None else 1, act, grad, float(negative_slope), float(scale), _lib.stream_ptr(x.device))
  return y


class FusedLeakyReLUFunctionBackward(Function):
  @staticmethod
  def forward(ctx, grad_output, out, negative_slope, scale):
    ctx.save_for_backward(out)
    ctx.negative_slope, ctx.scale = negative_slope, scale
    grad_input = _bias_act(grad_output, None, out, 3, 1, negative_slope, scale)
    dims = [0] + list(range(2, grad_input.ndim))
    return grad_input, grad_input.sum(dims).detach()

  @staticmethod
  def backward(ctx, gradgrad_input, gradgrad_bias):
    out, = ctx.saved_tensors
    return _bias_act(gradgrad_input, gradgrad_bias, out, 3, 1, ctx.negative_slope, ctx.scale), None, None, None


class FusedLeakyReLUFunction(Function):
  @staticmethod
  def forward(ctx, input, bias, negative_slope, scale):
    if not input.is_cuda:
      raise RuntimeError('fused_leaky_relu (score_sde_pytorch_b200): input must be a CUDA tensor (no CPU path)')
    out = _bias_act(input, bias, None, 3, 0, negative_slope, scale)
    ctx.save_for_backward(out)
    ctx.negative_slope, ctx.scale = negative_slope, scale
    return out

  @staticmethod
  def backward(ctx, grad_output):
    out, = ctx.saved_tensors
    grad_input, grad_bias = FusedLeakyReLUFunctionBackward.apply(grad_output, out, ctx.negative_slope, ctx.scale)
    return grad_input, grad_bias, None, None


def fused_leaky_relu(input, bias, negative_slope=0.2, scale=2 ** 0.5):
  if not input.is_cuda:
    raise RuntimeError('fused_leaky_relu (score_sde_pytorch_b200): input must be a CUDA tensor (no CPU path)')
  return FusedLeakyReLUFunction.apply(input, bias, negative_slope, scale)


class FusedLeakyReLU(nn.Module):
  def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5):
    super().__init__()
    self.bias = nn.Parameter(torch.zeros(channel))
    self.negative_slope = negative_slope
    self.scale = scale

  def forward(self, input):
    return fused_leaky_relu(input, self.bias, self.negative_slope, self.scale)
