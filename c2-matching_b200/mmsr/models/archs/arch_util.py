"""Building blocks shared by the archs (reference: mmsr/models/archs/arch_util.py; only the
pieces the restoration-forward path uses)."""
import torch
from torch import nn
from torch.nn import init


def default_init_weights(modules, scale=1.0):
    """Kaiming-normal (fan_in) x scale, zero bias — arch_util.py:40-61."""
    for root in modules if isinstance(modules, (list, tuple)) else [modules]:
        for m in root.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                init.kaiming_normal_(m.weight, a=0, mode='fan_in')
                with torch.no_grad():
                    m.weight.mul_(scale)
                    if m.bias is not None:
                        m.bias.zero_()


def srntt_init_weights(net, init_type='normal', init_gain=0.02):
    """N(0, gain) for every module whose class name contains Conv/Linear — arch_util.py:12-37.
    (DCN modules do not match and keep their own uniform init, as in the reference.)"""
    if init_type != 'normal':
        raise NotImplementedError(f'initialization method [{init_type}] is not implemented')
    for m in net.modules():
        cname = type(m).__name__
        if hasattr(m, 'weight') and ('Conv' in cname or 'Linear' in cname):
            init.normal_(m.weight.data, 0.0, init_gain)
            if getattr(m, 'bias', None) is not None:
                init.constant_(m.bias.data, 0.0)


class ResidualBlockNoBN(nn.Module):
    """x + conv2(relu(conv1(x))) * res_scale — arch_util.py:80-136 (state-dict keys conv1/conv2)."""

    def __init__(self, nf=64, res_scale=1, pytorch_init=False):
        super().__init__()
        self.res_scale = res_scale
        self.conv1 = Conv2d(nf, nf, 3, 1, 1, bias=True)
        self.conv2 = Conv2d(nf, nf, 3, 1, 1, bias=True)
        if not pytorch_init:
            default_init_weights([self.conv1, self.conv2], 0.1)

    def forward(self, x):
        y = self.conv2(torch.relu_(self.conv1(x)))
        return x + y if self.res_scale == 1 else x + y * self.res_scale


_warned_small = False


def fast_conv_enabled():
    """C2M_FAST_CONV=0 routes every plain convolution back to cuDNN (debug / A-B comparisons)."""
    import os
    return os.environ.get('C2M_FAST_CONV', '1') != '0'


def psa_path_ok(x, *convs, cat_first=32):
    """True if the tensor-core 3x3 kernel can take over for tensor `x` [B,C,H,W] and these convs.  `cat_first`: channel count of
    the FIRST input of the two-input (concatenating) convolutions on the path — the kernel needs a multiple of 32 there."""
    if not (fast_conv_enabled() and x.is_cuda and x.dtype == torch.float32 and not torch.is_grad_enabled()):
        return False
    from c2m_b200 import ops
    if not ops.conv3x3_supported(x.shape[2], x.shape[3]):
        # not silent: the tensor-core kernel needs one 18x10 halo tile; smaller maps run the plain modules (cuDNN, exact fp32)
        global _warned_small
        if not _warned_small:
            _warned_small = True
            import logging
            logging.getLogger('base').warning(
                f'c2m: feature map {x.shape[2]}x{x.shape[3]} is smaller than one halo tile (18x10): the plain 3x3 convolutions '
                'of this call run on nn.Conv2d (cuDNN, TF32 off), not on the tensor-core kernel')
        return False
    return all(_tc_conv(c) for c in convs) and cat_first % 32 == 0


def _tc_conv(c):
    """A convolution the tensor-core 3x3 kernel computes: 3x3 / stride 1 / pad 1 / dilation 1 / one group, on the GPU."""
    return (isinstance(c, nn.Conv2d) and c.kernel_size == (3, 3) and c.stride == (1, 1) and c.padding == (1, 1) and
            c.dilation == (1, 1) and c.groups == 1 and c.weight.is_cuda)


class Conv2d(nn.Conv2d):
    """nn.Conv2d (same parameters and state-dict keys) whose 3x3 / stride 1 / pad 1 instances run forward and backward
    on the tensor cores (c2m_b200.ops.conv3x3) under autograd, on the maps the inference path takes there: fp32 CUDA,
    at least 18x10, C2M_FAST_CONV not 0.  Everything else, inference under no_grad included, is nn.Conv2d."""

    def forward(self, x):
        if (torch.is_grad_enabled() and fast_conv_enabled() and _tc_conv(self) and self.padding_mode == 'zeros' and
                x.is_cuda and x.dtype == torch.float32 and x.dim() == 4):
            from c2m_b200 import ops
            if ops.conv3x3_supported(x.shape[2], x.shape[3]):
                return ops.conv3x3(x, self.weight, self.bias)
        return super().forward(x)


def conv_psa(conv, xp, act=None, **kw):
    """One nn.Conv2d (3x3/s1/p1) on a packed-split activation."""
    from c2m_b200 import ops
    return ops.conv3x3_psa(xp, conv.weight, conv.bias, act=act, **kw)


def resblocks_psa(body, hp, final_residual2=None):
    """Run a Sequential of ResidualBlockNoBN on a packed-split activation (PSA) with the tensor-core
    3x3 kernel: x + conv2(relu(conv1(x))) per block, two launches per block, no fp32 round trip.
    `final_residual2` is added in the last block's epilogue (the `body(h) + x` skip of
    ref_restoration_arch.py:158,171,184).  Three PSA buffers are cycled."""
    from c2m_b200 import ops
    bufs = [hp, ops.PSA.empty(hp.B, hp.C, hp.H, hp.W, hp.hi.device), ops.PSA.empty(hp.B, hp.C, hp.H, hp.W, hp.hi.device)]
    cur = 0
    n = len(body)
    for i, blk in enumerate(body):
        if blk.res_scale != 1:
            raise NotImplementedError('res_scale != 1 is not used by C2-Matching')
        t, nxt = bufs[(cur + 1) % 3], bufs[(cur + 2) % 3]
        ops.conv3x3_psa(bufs[cur], blk.conv1.weight, blk.conv1.bias, act='relu', out=t)
        ops.conv3x3_psa(t, blk.conv2.weight, blk.conv2.bias, act=None, residual=bufs[cur],
                        residual2=final_residual2 if i == n - 1 else None, out=nxt)
        cur = (cur + 2) % 3
    return bufs[cur]


def body_forward(body, h, skip=None):
    """body(h) (+ skip) on fp32 tensors: tensor-core path when supported, else the plain modules."""
    from c2m_b200 import ops
    if all(isinstance(b, ResidualBlockNoBN) for b in body) and psa_path_ok(h, body[0].conv1, body[0].conv2):
        out = resblocks_psa(body, ops.psa_from_f32(h))
        return ops.psa_to_f32(out, add=skip)
    y = body(h)
    return y if skip is None else y + skip


def attach_psa(t, psa):
    """Remember the packed-split twin of an fp32 feature tensor (consumed by the next fast conv)."""
    try:
        t._c2m_psa = psa
    except Exception:
        pass
    return t


def psa_of(t):
    """Packed-split version of fp32 tensor `t` (reusing the twin a producer attached, if any)."""
    from c2m_b200 import ops
    p = getattr(t, '_c2m_psa', None)
    if p is not None and p.shape == tuple(t.shape):
        return p
    return ops.psa_from_f32(t)


def make_layer(block, n_blocks, **kwargs):
    return nn.Sequential(*[block(**kwargs) for _ in range(n_blocks)])


def tensor_shift(x, shift=(2, 2), fill_val=0):
    """Shift [b,h,w,c] down/right with constant fill — arch_util.py:291-315.  Kept for API
    parity; the H100 path builds all shifted offsets in one kernel (csrc/offsets.cu)."""
    sh, sw = shift
    if sh < 0 or sw < 0:
        raise NotImplementedError
    out = torch.full_like(x, fill_val)
    h, w = x.shape[1:3]
    out[:, sh:, sw:, :] = x[:, :h - sh, :w - sw, :]
    return out
