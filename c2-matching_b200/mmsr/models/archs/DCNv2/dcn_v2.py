"""DCNv2 module layer with the reference's class names and state-dict keys
(mmsr/models/archs/DCNv2/dcn_v2.py) on top of the drop-in `_ext`: the deformable convolutions
(`DCNv2`, `DCN`, `DCN_sep`, `DCN_sep_pre_multi_offset`) and the deformable PS-ROI pooling modules
(`DCNv2Pooling`, `DCNPooling`), forward and backward through `_ext`.

`DCN_sep_pre_multi_offset` — the only variant C2-Matching instantiates
(ref_restoration_arch.py:5) — runs its whole tail (offset add + reorder, sigmoid, deformable
sampling, contraction, bias, optional LeakyReLU) in ONE kernel and drops the reference's
host-synchronising `offset_mean > 100` check (dcn_v2.py:247-250) unless `debug_offset_check`."""
import logging
import math
import os

import _ext as _backend
import torch
from torch import nn
from torch.nn.modules.utils import _pair

from c2m_b200 import ops as _ops
from ..arch_util import Conv2d

logger = logging.getLogger('base')


class _DCNv2(torch.autograd.Function):
    """The reference's autograd Function (dcn_v2.py:16-50): forward and backward both cross the
    `_ext` boundary."""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups):
        ctx.geom = (tuple(weight.shape[2:4]), _pair(stride), _pair(padding), _pair(dilation), deformable_groups)
        (kh, kw), (sh, sw), (ph, pw), (dh, dw), dg = ctx.geom
        out = _backend.dcn_v2_forward(input, weight, bias, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, dg)
        ctx.save_for_backward(input, offset, mask, weight, bias)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_output):
        input, offset, mask, weight, bias = ctx.saved_tensors
        (kh, kw), (sh, sw), (ph, pw), (dh, dw), dg = ctx.geom
        gi, go, gm, gw, gb = _backend.dcn_v2_backward(input, weight, bias, offset, mask, grad_output.contiguous(),
                                                      kh, kw, sh, sw, ph, pw, dh, dw, dg)
        return gi, go, gm, gw, gb, None, None, None, None


dcn_v2_conv = _DCNv2.apply


class DCNv2(nn.Module):
    """dcn_v2.py:56-95: owns `weight` [Cout,Cin,kh,kw] and `bias`."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation = _pair(padding), _pair(dilation)
        self.deformable_groups = deformable_groups
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, *self.kernel_size))
        self.bias = nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1.0 / math.sqrt(self.in_channels * self.kernel_size[0] * self.kernel_size[1])
        with torch.no_grad():
            self.weight.uniform_(-stdv, stdv)
            self.bias.zero_()

    def _check(self, offset, mask):
        taps = self.deformable_groups * self.kernel_size[0] * self.kernel_size[1]
        assert offset.shape[1] == 2 * taps and mask.shape[1] == taps

    def forward(self, input, offset, mask):
        self._check(offset, mask)
        return dcn_v2_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups)


class _WithOffsetConv(DCNv2):
    """Adds the zero-initialised `conv_offset_mask` (3*dg*kh*kw channels) the DCN variants share."""

    def __init__(self, *args, extra_offset_mask=None, **kwargs):
        super().__init__(*args, **kwargs)
        if extra_offset_mask is not None:
            self.extra_offset_mask = extra_offset_mask
        self.conv_offset_mask = Conv2d(self.in_channels, 3 * self.deformable_groups * self.kernel_size[0] *
                                       self.kernel_size[1], self.kernel_size, self.stride, self.padding, bias=True)
        self.init_offset()

    def init_offset(self):
        with torch.no_grad():
            self.conv_offset_mask.weight.zero_()
            self.conv_offset_mask.bias.zero_()

    def _offset_mask(self, feat):
        out = self.conv_offset_mask(feat)
        n = out.shape[1] // 3
        return out[:, :2 * n], torch.sigmoid(out[:, 2 * n:])


class DCN(_WithOffsetConv):
    """dcn_v2.py:98-133."""

    def forward(self, input):
        offset, mask = self._offset_mask(input)
        return dcn_v2_conv(input, offset.contiguous(), mask, self.weight, self.bias, self.stride, self.padding,
                           self.dilation, self.deformable_groups)


class DCN_sep(_WithOffsetConv):
    """dcn_v2.py:136-184: offsets/masks predicted from a second feature map."""

    def __init__(self, *args, extra_offset_mask=True, **kwargs):
        super().__init__(*args, extra_offset_mask=extra_offset_mask, **kwargs)

    def forward(self, x):
        feat = x
        if self.extra_offset_mask:
            x, feat = x[0], x[1]
        offset, mask = self._offset_mask(feat)
        return dcn_v2_conv(x, offset.contiguous(), mask, self.weight, self.bias, self.stride, self.padding,
                           self.dilation, self.deformable_groups)


class DCN_sep_pre_multi_offset(_WithOffsetConv):
    """dcn_v2.py:187-253: learned offsets are residuals on top of the precomputed non-local
    offsets from the correspondence search."""

    debug_offset_check = False   # True restores the reference's (host-syncing) warning

    def __init__(self, *args, extra_offset_mask=True, **kwargs):
        super().__init__(*args, extra_offset_mask=extra_offset_mask, **kwargs)

    def forward(self, x, pre_offset, lrelu_slope=1.0, channels_last_out=False):
        feat = x
        if self.extra_offset_mask:
            x, feat = x[0], x[1]
        return self.fused_tail(x, self.conv_offset_mask(feat), pre_offset, lrelu_slope, channels_last_out)

    def fused_tail(self, x, om, pre_offset, lrelu_slope=1.0, channels_last_out=False, want_psa=False):
        """Everything after the conv_offset_mask convolution (dcn_v2.py:230-253), one kernel.
        `om`: raw conv_offset_mask output [B, 3*dg*9, H, W] fp32.  With want_psa the result is
        returned in the packed-split layout (tensor-core kernel only)."""
        if self.stride != (1, 1) or self.dilation != (1, 1):
            raise NotImplementedError('fused pre-offset DCN supports stride 1 / dilation 1 (all C2-Matching uses)')
        tc = (self.kernel_size == (3, 3) and self.padding == (1, 1) and lrelu_slope in (1.0, 0.1) and
              os.environ.get('C2M_DCN_TC', '1') != '0' and
              _ops.dcn_tc_supported(self.in_channels, self.out_channels, self.deformable_groups))
        grad = torch.is_grad_enabled() and (getattr(om, 'requires_grad', False) or getattr(x, 'requires_grad', False) or
                                            self.weight.requires_grad)
        if isinstance(om, _ops.OctF32) and (self.debug_offset_check or grad or not tc):
            om = om.nchw()       # octet-planar offsets are only understood by the tensor-core kernel
        if isinstance(x, _ops.PSA) and (grad or not tc):
            x = _ops.psa_to_f32(x)
        if self.debug_offset_check:
            mean = om[:, :om.shape[1] // 3 * 2].abs().mean()
            if mean > 100:
                logger.warning(f'Offset mean is {mean}, larger than 100.')
        if grad:
            # training: the reference's differentiable formulation (dcn_v2.py:231-253) over dcn_v2_conv
            pre = pre_offset.materialize() if hasattr(pre_offset, 'materialize') else pre_offset
            n = om.shape[1] // 3
            reord = torch.stack((pre[..., 1], pre[..., 0]), dim=2).flatten(1, 2).repeat(1, self.deformable_groups, 1, 1)
            offset, mask = om[:, :2 * n] + reord, torch.sigmoid(om[:, 2 * n:])
            # The tensor-core backward sums grad_input with atomics (every other gradient has a fixed order), and with
            # grad_input it is slower than `_ext`'s on the 256-channel layer (DESIGN.md §4, K8): both cases keep `_ext`.
            x_excluded = x.requires_grad and (_ops.deterministic() or self.in_channels >= 256)
            if tc and not x_excluded and _ops.dcn_tc_backward_supported(self.in_channels, self.out_channels,
                                                                        self.deformable_groups, *x.shape[2:]):
                out = _ops.dcn_v2_tc(x, offset, mask, self.weight, self.bias, self.deformable_groups)
            else:
                out = dcn_v2_conv(x, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                                  self.deformable_groups)
            out = out if lrelu_slope == 1.0 else torch.nn.functional.leaky_relu(out, lrelu_slope)
            return _ops.psa_from_f32(out) if want_psa else out
        idx = getattr(pre_offset, 'max_idx', None)
        kw = dict(idx=idx, pre_scale=pre_offset.scale, ref_gw=pre_offset.ref_gw) if idx is not None else \
            dict(pre_offset=pre_offset)          # ScaleOffsets handle: no offset pyramid in HBM
        if tc:
            return _ops.dcn_v2_fused_tc(x, om, self.weight, self.bias, self.deformable_groups, lrelu=lrelu_slope == 0.1,
                                        psa_out=want_psa, out_f32=not want_psa, channels_last_out=channels_last_out, **kw)
        out = _ops.dcn_v2_fused_forward(x, om, self.weight, self.bias, self.deformable_groups,
                                        lrelu_slope=lrelu_slope, channels_last_out=channels_last_out, **kw)
        return _ops.psa_from_f32(out) if want_psa else out


class _DCNv2Pooling(torch.autograd.Function):
    """The reference's pooling Function (dcn_v2.py:256-307): forward and backward both cross the `_ext` boundary;
    gradients flow to `input` and `offset` (the translations), not to `rois`."""

    @staticmethod
    def forward(ctx, input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1,
                part_size=None, sample_per_part=4, trans_std=.0):
        ctx.args = (int(no_trans), spatial_scale, output_dim, group_size, pooled_size,
                    pooled_size if part_size is None else part_size, sample_per_part, trans_std)
        output, output_count = _backend.dcn_v2_psroi_pooling_forward(input, rois, offset, *ctx.args)
        ctx.save_for_backward(input, rois, offset, output_count)
        return output

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_output):
        input, rois, offset, output_count = ctx.saved_tensors
        grad_input, grad_offset = _backend.dcn_v2_psroi_pooling_backward(grad_output.contiguous(), input, rois, offset,
                                                                         output_count, *ctx.args)
        return grad_input, None, grad_offset, None, None, None, None, None, None, None, None


dcn_v2_pooling = _DCNv2Pooling.apply


class DCNv2Pooling(nn.Module):
    """dcn_v2.py:313-341: pools with the given per-ROI translations `offset` [R, 2K, part, part] (ignored when
    no_trans)."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0):
        super().__init__()
        self.spatial_scale = spatial_scale
        self.pooled_size = pooled_size
        self.output_dim = output_dim
        self.no_trans = no_trans
        self.group_size = group_size
        self.part_size = pooled_size if part_size is None else part_size
        self.sample_per_part = sample_per_part
        self.trans_std = trans_std

    def _pool(self, input, rois, offset, no_trans):
        return dcn_v2_pooling(input, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim, no_trans,
                              self.group_size, self.part_size, self.sample_per_part, self.trans_std)

    def forward(self, input, rois, offset):
        assert input.shape[1] == self.output_dim
        if self.no_trans:
            offset = input.new()
        return self._pool(input, rois, offset, self.no_trans)


class DCNPooling(DCNv2Pooling):
    """dcn_v2.py:344-411: unless no_trans, predicts one translation and one sigmoid modulation per bin from a first,
    untranslated pooling through `offset_mask_fc` (last layer zero-initialised, so training starts from plain pooling),
    then pools again with the translations and multiplies by the modulation."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0, deform_fc_dim=1024):
        super().__init__(spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part,
                         trans_std)
        self.deform_fc_dim = deform_fc_dim
        if not no_trans:
            bins = self.pooled_size * self.pooled_size
            self.offset_mask_fc = nn.Sequential(
                nn.Linear(bins * self.output_dim, self.deform_fc_dim), nn.ReLU(inplace=True),
                nn.Linear(self.deform_fc_dim, self.deform_fc_dim), nn.ReLU(inplace=True),
                nn.Linear(self.deform_fc_dim, bins * 3))
            with torch.no_grad():
                self.offset_mask_fc[4].weight.zero_()
                self.offset_mask_fc[4].bias.zero_()

    def forward(self, input, rois):
        offset = input.new()
        if self.no_trans:
            return self._pool(input, rois, offset, self.no_trans)
        n = rois.shape[0]
        roi = self._pool(input, rois, offset, True)
        offset_mask = self.offset_mask_fc(roi.view(n, -1)).view(n, 3, self.pooled_size, self.pooled_size)
        o1, o2, mask = torch.chunk(offset_mask, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        return self._pool(input, rois, offset, self.no_trans) * torch.sigmoid(mask)
