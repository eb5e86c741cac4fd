"""Drop-in replacement for the reference's compiled `deform_conv_cuda` extension
(mmsr/models/archs/dcn/src/deform_conv_cuda.cpp:681-695): the same five functions with the same positional
arguments and the same in-place contract on the result tensors the caller passes in.  The arithmetic runs in
libc2m_sm100.so (c2m_deform_conv_*, include/c2m_sm100.h) through c2m_b200.ops.

- The forwards OVERWRITE `output`; the modulated one adds `bias` only when `with_bias` is set.
- `deform_conv_backward_input_cuda` ADDS into `gradInput` and OVERWRITES `gradOffset`.
- `deform_conv_backward_parameters_cuda` does `gradWeight += scale * sum`.
- `modulated_deform_conv_cuda_backward` ADDS into `grad_input`, `grad_weight` and `grad_bias` and OVERWRITES
  `grad_offset` and `grad_mask`.
- `columns` and `ones` are the reference's scratch buffers: accepted and not used.
- `im2col_step` changes no result (the batch is a grid dimension of every kernel); only the check that it divides
  the batch is kept.
fp32 and fp64; other dtypes, CPU tensors and input that is not 4-D raise, and so do launch errors."""
from c2m_b200 import ops as _ops


def _check_4d(input):
    if input.dim() != 4:
        raise RuntimeError(f'4D input tensor [B, C, H, W] expected, got {input.dim()}D (3-D input is not supported)')


def _check_step(input, im2col_step):
    step = min(im2col_step, input.shape[0])
    assert input.shape[0] % step == 0, 'im2col step must divide batchsize'


def _check_weight(weight):
    if weight.dim() != 4:
        raise RuntimeError(f'4D weight tensor (nOutputPlane,nInputPlane,kH,kW) expected, but got: {weight.dim()}')
    if not weight.is_contiguous():
        raise RuntimeError('weight tensor has to be contiguous')


def _check_contiguous(input, weight):
    if not input.is_contiguous():
        raise RuntimeError('input tensor has to be contiguous')
    if not weight.is_contiguous():
        raise RuntimeError('weight tensor has to be contiguous')


def deform_conv_forward_cuda(input, weight, offset, output, columns, ones, kW, kH, dW, dH, padW, padH, dilationW,
                             dilationH, group, deformable_group, im2col_step):
    _check_4d(input)
    _check_weight(weight)
    _check_step(input, im2col_step)
    out = _ops.deform_conv_forward(input, weight, offset, None, None, kH, kW, dH, dW, padH, padW, dilationH,
                                   dilationW, group, deformable_group)
    output.copy_(out)
    return 1


def deform_conv_backward_input_cuda(input, offset, gradOutput, gradInput, gradOffset, weight, columns, kW, kH, dW,
                                    dH, padW, padH, dilationW, dilationH, group, deformable_group, im2col_step):
    _check_4d(input)
    _check_weight(weight)
    _check_step(input, im2col_step)
    gi, go, _, _, _ = _ops.deform_conv_backward(input, weight, offset, None, gradOutput, kH, kW, dH, dW, padH, padW,
                                                dilationH, dilationW, group, deformable_group, need_weight=False)
    gradInput.add_(gi)
    gradOffset.copy_(go)
    return 1


def deform_conv_backward_parameters_cuda(input, offset, gradOutput, gradWeight, columns, ones, kW, kH, dW, dH, padW,
                                         padH, dilationW, dilationH, group, deformable_group, scale, im2col_step):
    _check_4d(input)
    _check_weight(gradWeight)
    _check_step(input, im2col_step)
    _, _, _, gw, _ = _ops.deform_conv_backward(input, gradWeight, offset, None, gradOutput, kH, kW, dH, dW, padH, padW,
                                               dilationH, dilationW, group, deformable_group, need_input=False)
    gradWeight.add_(gw, alpha=scale)
    return 1


def modulated_deform_conv_cuda_forward(input, weight, bias, ones, offset, mask, output, columns, kernel_h, kernel_w,
                                       stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group,
                                       deformable_group, with_bias):
    _check_4d(input)
    _check_contiguous(input, weight)
    out = _ops.deform_conv_forward(input, weight, offset, mask, bias if with_bias else None, kernel_h, kernel_w,
                                   stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group, deformable_group)
    output.copy_(out)


def modulated_deform_conv_cuda_backward(input, weight, bias, ones, offset, mask, columns, grad_input, grad_weight,
                                        grad_bias, grad_offset, grad_mask, grad_output, kernel_h, kernel_w, stride_h,
                                        stride_w, pad_h, pad_w, dilation_h, dilation_w, group, deformable_group,
                                        with_bias):
    _check_4d(input)
    _check_contiguous(input, weight)
    gi, go, gm, gw, gb = _ops.deform_conv_backward(input, weight, offset, mask, grad_output, kernel_h, kernel_w,
                                                   stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group,
                                                   deformable_group)
    grad_input.add_(gi)
    grad_weight.add_(gw)
    if with_bias:
        grad_bias.add_(gb)
    grad_offset.copy_(go)
    grad_mask.copy_(gm)
