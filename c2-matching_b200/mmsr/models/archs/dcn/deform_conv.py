"""Deformable convolution v1 and modulated (v2) with the reference's public surface
(mmsr/models/archs/dcn/deform_conv.py): the Functions `deform_conv` / `modulated_deform_conv` and the modules
`DeformConv`, `DeformConvPack`, `ModulatedDeformConv`, `ModulatedDeformConvPack` with the same constructor arguments,
parameter shapes, initialisation and state-dict keys (`weight`, `bias`, `conv_offset.*`, `conv_offset_mask.*`).
They call the drop-in `deform_conv_cuda` (libc2m_sm100 kernels, fp32 and fp64, any conv / deformable groups).

Deliberate differences from the reference:
- `DeformConvFunction.backward` returns one gradient per forward input (9); the reference returns 8, which current
  torch rejects.
- fp16 raises (the reference's im2col dispatched half).
- Input that is not 4-D raises in both Functions (the reference's v1 Function already rejects it).
- Output channels not divisible by `groups` raise a clear error instead of failing in a `view`.
- Launch errors raise instead of being printed.
- `ModulatedDeformConvPack` computes the offset mean for its `> 100` warning (a host synchronisation) only with
  `debug_offset_check=True`.
The modulated Function keeps the reference's int-only stride, padding and dilation (each passed for both axes)."""
import logging
import math

import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from . import deform_conv_cuda as _cuda

logger = logging.getLogger('base')


def _require_4d(input):
    if input.dim() != 4:
        raise ValueError(f'Expected 4D tensor as input, got {input.dim()}D tensor instead.')


def _require_cuda(input):
    if not input.is_cuda:
        raise NotImplementedError('deformable convolution runs on CUDA tensors only')


def _step(input, im2col_step):
    """The reference's im2col chunk (no effect on the result here); it must divide the batch."""
    step = min(im2col_step, input.shape[0])
    assert input.shape[0] % step == 0, 'im2col step must divide batchsize'
    return step


def _scratch(input):
    return input.new_empty(0)


class DeformConvFunction(Function):
    """DCNv1: output = sum over taps of weight * bilinear(input, tap position + offset), per conv group."""

    @staticmethod
    def forward(ctx, input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1,
                im2col_step=64):
        _require_4d(input)
        (sh, sw), (ph, pw), (dh, dw) = ctx.geom = (_pair(stride), _pair(padding), _pair(dilation))
        ctx.groups, ctx.deformable_groups, ctx.im2col_step = groups, deformable_groups, im2col_step
        out_hw = []
        for n, k, s, p, d in zip(input.shape[2:], weight.shape[2:], (sh, sw), (ph, pw), (dh, dw)):
            out_hw.append((n + 2 * p - (d * (k - 1) + 1)) // s + 1)
        size = (input.shape[0], weight.shape[0], *out_hw)
        if min(size) < 1:
            raise ValueError('convolution input is too small (output would be {})'.format('x'.join(map(str, size))))
        _require_cuda(input)
        output = input.new_empty(size)
        _cuda.deform_conv_forward_cuda(input, weight, offset, output, _scratch(input), _scratch(input),
                                       weight.shape[3], weight.shape[2], sw, sh, pw, ph, dw, dh, groups,
                                       deformable_groups, _step(input, im2col_step))
        ctx.save_for_backward(input, offset, weight)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        input, offset, weight = ctx.saved_tensors
        _require_cuda(grad_output)
        (sh, sw), (ph, pw), (dh, dw) = ctx.geom
        kh, kw = weight.shape[2:]
        step = _step(input, ctx.im2col_step)
        grad_output = grad_output.contiguous()
        geom = (kw, kh, sw, sh, pw, ph, dw, dh, ctx.groups, ctx.deformable_groups)
        grad_input = grad_offset = grad_weight = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            grad_input, grad_offset = torch.zeros_like(input), torch.zeros_like(offset)
            _cuda.deform_conv_backward_input_cuda(input, offset, grad_output, grad_input, grad_offset, weight,
                                                  _scratch(input), *geom, step)
        if ctx.needs_input_grad[2]:
            grad_weight = torch.zeros_like(weight)
            _cuda.deform_conv_backward_parameters_cuda(input, offset, grad_output, grad_weight, _scratch(input),
                                                       _scratch(input), *geom, 1, step)
        # one entry per forward input: input, offset, weight, stride, padding, dilation, groups, dg, im2col_step
        return grad_input, grad_offset, grad_weight, None, None, None, None, None, None


class ModulatedDeformConvFunction(Function):
    """Modulated (DCNv2): as DeformConvFunction with each sample scaled by `mask`, plus an optional bias.  stride,
    padding and dilation are ints, applied to both axes."""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                deformable_groups=1):
        _require_4d(input)
        _require_cuda(input)
        ctx.stride, ctx.padding, ctx.dilation = stride, padding, dilation
        ctx.groups, ctx.deformable_groups = groups, deformable_groups
        ctx.with_bias = bias is not None
        if bias is None:
            bias = input.new_empty(1)       # placeholder, as in the reference; not read
        if input.requires_grad or offset.requires_grad or mask.requires_grad or weight.requires_grad:
            ctx.save_for_backward(input, offset, mask, weight, bias)
        kh, kw = weight.shape[2:4]
        ho = (input.shape[2] + 2 * padding - (dilation * (kh - 1) + 1)) // stride + 1
        wo = (input.shape[3] + 2 * padding - (dilation * (kw - 1) + 1)) // stride + 1
        output = input.new_empty(input.shape[0], weight.shape[0], ho, wo)
        _cuda.modulated_deform_conv_cuda_forward(input, weight, bias, _scratch(input), offset, mask, output,
                                                 _scratch(input), kh, kw, stride, stride, padding, padding, dilation,
                                                 dilation, groups, deformable_groups, ctx.with_bias)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        _require_cuda(grad_output)
        input, offset, mask, weight, bias = ctx.saved_tensors
        grads = [torch.zeros_like(t) for t in (input, offset, mask, weight, bias)]
        grad_input, grad_offset, grad_mask, grad_weight, grad_bias = grads
        _cuda.modulated_deform_conv_cuda_backward(
            input, weight, bias, _scratch(input), offset, mask, _scratch(input), grad_input, grad_weight, grad_bias,
            grad_offset, grad_mask, grad_output.contiguous(), weight.shape[2], weight.shape[3], ctx.stride,
            ctx.stride, ctx.padding, ctx.padding, ctx.dilation, ctx.dilation, ctx.groups, ctx.deformable_groups,
            ctx.with_bias)
        return (grad_input, grad_offset, grad_mask, grad_weight, grad_bias if ctx.with_bias else None,
                None, None, None, None, None)


deform_conv = DeformConvFunction.apply
modulated_deform_conv = ModulatedDeformConvFunction.apply


def _init_weight(weight, in_channels, kernel_size):
    """uniform(-1/sqrt(n), 1/sqrt(n)) with n = in_channels * kh * kw (all input channels, not per group)."""
    bound = 1. / math.sqrt(in_channels * kernel_size[0] * kernel_size[1])
    weight.data.uniform_(-bound, bound)


def _zero_conv(in_channels, out_channels, kernel_size, stride, padding):
    """The offset (/ mask) predictor of the Pack modules, zero-initialised: they start as plain convolutions."""
    conv = nn.Conv2d(in_channels, out_channels, kernel_size=kernel_size, stride=_pair(stride),
                     padding=_pair(padding), bias=True)
    conv.weight.data.zero_()
    conv.bias.data.zero_()
    return conv


class DeformConv(nn.Module):
    """DCNv1 layer: `weight` [out_channels, in_channels / groups, kh, kw]; no bias (bias=True is refused)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=False):
        super().__init__()
        assert not bias
        assert in_channels % groups == 0, f'in_channels {in_channels} cannot be divisible by groups {groups}'
        assert out_channels % groups == 0, f'out_channels {out_channels} cannot be divisible by groups {groups}'
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation = _pair(padding), _pair(dilation)
        self.groups, self.deformable_groups = groups, deformable_groups
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, *self.kernel_size))
        self.reset_parameters()

    def reset_parameters(self):
        _init_weight(self.weight, self.in_channels, self.kernel_size)

    def forward(self, x, offset):
        return deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups,
                           self.deformable_groups)


class DeformConvPack(DeformConv):
    """DeformConv that predicts its offsets from its input with `conv_offset` (2 * dg * kh * kw channels)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = _zero_conv(self.in_channels, 2 * self.deformable_groups * self.kernel_size[0] *
                                      self.kernel_size[1], self.kernel_size, self.stride, self.padding)

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        return super().forward(x, self.conv_offset(x))


class ModulatedDeformConv(nn.Module):
    """Modulated layer: `weight` [out_channels, in_channels / groups, kh, kw] and `bias` (None when bias=False).
    stride, padding and dilation are ints."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride, self.padding, self.dilation = stride, padding, dilation
        self.groups, self.deformable_groups = groups, deformable_groups
        self.with_bias = bias
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, *self.kernel_size))
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        _init_weight(self.weight, self.in_channels, self.kernel_size)
        if self.bias is not None:
            self.bias.data.zero_()

    def forward(self, x, offset, mask):
        return modulated_deform_conv(x, offset, mask, self.weight, self.bias, self.stride, self.padding,
                                     self.dilation, self.groups, self.deformable_groups)


class ModulatedDeformConvPack(ModulatedDeformConv):
    """ModulatedDeformConv that predicts offsets and mask with `conv_offset_mask` (3 * dg * kh * kw channels: two
    offset thirds, then the mask logits, passed through a sigmoid).  With extra_offset_mask the input is
    [x, features] and the prediction reads `features`.  debug_offset_check=True restores the reference's warning
    when the mean |offset| exceeds 100 (it synchronises with the host)."""

    def __init__(self, *args, extra_offset_mask=False, debug_offset_check=False, **kwargs):
        super().__init__(*args, **kwargs)
        self.extra_offset_mask = extra_offset_mask
        self.debug_offset_check = debug_offset_check
        self.conv_offset_mask = _zero_conv(self.in_channels, 3 * self.deformable_groups * self.kernel_size[0] *
                                           self.kernel_size[1], self.kernel_size, self.stride, self.padding)

    def init_offset(self):
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()

    def forward(self, x):
        x, feat = (x[0], x[1]) if self.extra_offset_mask else (x, x)
        n = self.conv_offset_mask.out_channels // 3
        om = self.conv_offset_mask(feat)
        offset, mask = om[:, :2 * n], torch.sigmoid(om[:, 2 * n:])
        if self.debug_offset_check:
            offset_mean = torch.mean(torch.abs(offset))
            if offset_mean > 100:
                logger.warning(f'Offset mean is {offset_mean}, larger than 100.')
        return super().forward(x, offset.contiguous(), mask.contiguous())
