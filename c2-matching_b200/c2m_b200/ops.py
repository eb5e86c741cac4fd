"""Torch-facing wrappers over the C ABI.  Inputs must be CUDA fp32 tensors (fp32 or fp64 for the PS-ROI pooling and
grouped deformable convolution entries); outputs are
allocated here with torch (caller-owned in ABI terms) and raw pointers + the current stream
are handed to the library."""
import ctypes
import math
import os
import weakref

import torch

from . import _lib
from ._lib import DcnShape

_ws_cache = {}
_DTYPE_SFX = {torch.float32: 'f32', torch.float64: 'f64'}      # entry-point suffix of each dtype


def _require_cuda(name, t, dtype=torch.float32):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f'{name} must be a Tensor')
    if not t.is_cuda:
        # reference: AT_ERROR("Not implemented on the CPU") — DCNv2/src/dcn_v2.h:38
        raise RuntimeError(f'{name} must be a CUDA tensor (Not implemented on the CPU)')
    if t.dtype != dtype:
        raise RuntimeError(f'{name} must be {dtype}, got {t.dtype}')


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _call(name, *args, device=None):
    """Runs the entry point `name` with `device` current (None: as it is) on that device's current stream, which goes
    in as the last argument: tensors go in as their data pointers, None, numbers and ctypes structs as given.  The
    symbol is looked up on every call, so that a wrapper set on the library object sees it; a nonzero status raises
    C2MError."""
    if device is not None:
        with torch.cuda.device(device):
            return _call(name, *args)
    fn = getattr(_lib.lib(), name)
    _lib.check(fn(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args], _stream()), name)


def _size(name, *args):
    """The byte count the size query `name` returns; 0 (a bad shape) raises C2MError."""
    return _lib.check_size(getattr(_lib.lib(), name)(*args), name)


def _memory_format(channels_last):
    return torch.channels_last if channels_last else torch.contiguous_format


def _empty_f32(B, C, H, W, device, channels_last=False):
    return torch.empty(B, C, H, W, dtype=torch.float32, device=device, memory_format=_memory_format(channels_last))


def _one_or_both(psa, f32):
    """(psa, f32) when both outputs were made, else the one that was."""
    if psa is not None and f32 is not None:
        return psa, f32
    return psa if psa is not None else f32


def launch_count():
    return int(_lib.lib().c2m_launch_count())


def profile_enable(on=True):
    _lib.check(_lib.lib().c2m_profile_enable(int(bool(on))), 'c2m_profile_enable')


PROF_KERNELS = {'corr_search': 0, 'conv3x3': 1, 'dcn': 2, 'dcn_dgrad': 3, 'dcn_wgrad': 4, 'conv3x3_wgrad': 5}


def profile_collect(kernel):
    """{'ms', 'launches', 'flops', 'bytes'} of one kernel class since the last collect."""
    ms, n, fl, by = ctypes.c_float(0), ctypes.c_int(0), ctypes.c_double(0), ctypes.c_double(0)
    _lib.check(_lib.lib().c2m_profile_collect(PROF_KERNELS[kernel], ctypes.byref(ms), ctypes.byref(n),
                                              ctypes.byref(fl), ctypes.byref(by)), 'c2m_profile_collect')
    return {'ms': float(ms.value), 'launches': int(n.value), 'flops': float(fl.value), 'bytes': float(by.value)}


def _workspace(nbytes, device):
    """Per-(device, stream) scratch, grown on demand.  Re-entrant across DataParallel threads:
    each replica runs on its own device."""
    key = (device.index, _stream())
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


# ------------------------------------------------------------------------------------------------
# Ordered input gradients.  With torch.use_deterministic_algorithms(True) (warn_only or not) the three backward entries
# below compute grad_input with the c2m_*_det entry points, which add every element's contributions in one fixed order
# (include/c2m_sm100.h, "ordered input gradients"); otherwise the atomic scatters run.
DET_WORKSPACE_CAP = 1 << 30      # planes per pass are capped so that the workspace stays near this size (>= one plane)
det_workspace_peak = 0           # largest ordered-gather workspace allocated so far, in bytes (tools/ read and reset it)


def deterministic():
    return torch.are_deterministic_algorithms_enabled()


def _det_workspace(query, shape, nplanes, device):
    """Workspace for an ordered gather: as many planes per pass as fit in DET_WORKSPACE_CAP, at least one.  Call with
    `device` current (the size query asks CUB, which reads the current device)."""
    global det_workspace_peak
    one = _size(query, shape, 1)
    planes = max(1, min(nplanes, DET_WORKSPACE_CAP // one))
    nbytes = _size(query, shape, planes) if planes > 1 else one
    det_workspace_peak = max(det_workspace_peak, int(nbytes))
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


def _col2im(sfx, gcol, offset, mask, s, x):
    """grad_input of the deformable convolution from gcol: the ordered gather when deterministic algorithms are on,
    else the atomic scatter into zeros."""
    if deterministic():
        grad_input = torch.empty_like(x)
        ws = _det_workspace('c2m_dcn_col2im_det_workspace_bytes', s, s.B * s.dg, x.device)
        _call(f'c2m_deform_conv_col2im_det_{sfx}', gcol, offset, mask, s, grad_input, ws, ws.numel())
        return grad_input
    grad_input = torch.zeros_like(x)
    _call(f'c2m_deform_conv_col2im_{sfx}', gcol, offset, mask, s, grad_input)
    return grad_input


def corr_argmax(feat_in, feat_ref, patch_size=3, input_stride=1, ref_stride=1, is_norm=True,
                norm_input=False, l2norm=False, force_generic=False):
    """Batched correlation + argmax.  feat_in [B,C,h,w], feat_ref [B,C,hr,wr] ->
    (idx int64 [B,h',w'], val fp32 [B,h',w']).  See include/c2m_sm100.h."""
    _require_cuda('feat_input', feat_in)
    _require_cuda('feat_ref', feat_ref)
    if feat_in.dim() != 4 or feat_ref.dim() != 4:
        raise RuntimeError('corr_argmax expects [B,C,h,w] tensors')
    if feat_in.shape[:2] != feat_ref.shape[:2]:
        raise RuntimeError(f'batch/channel mismatch: {tuple(feat_in.shape)} vs {tuple(feat_ref.shape)}')
    feat_in = feat_in.contiguous()
    feat_ref = feat_ref.contiguous()
    B, C, h, w = feat_in.shape
    hr, wr = feat_ref.shape[2:]
    with torch.cuda.device(feat_in.device):
        need = _size('c2m_corr_workspace_bytes', B, C, h, w, hr, wr, patch_size, input_stride, ref_stride)
        ws = _workspace(need, feat_in.device)
        gh, gw = (h - patch_size) // input_stride + 1, (w - patch_size) // input_stride + 1
        idx = torch.empty(B, gh, gw, dtype=torch.int64, device=feat_in.device)
        val = torch.empty(B, gh, gw, dtype=torch.float32, device=feat_in.device)
        _call('c2m_corr_argmax_f32', feat_in, feat_ref, B, C, h, w, hr, wr, patch_size, input_stride, ref_stride,
              int(is_norm), int(norm_input), int(l2norm), 1 if force_generic else 0, idx, val, ws, ws.numel())
    return idx, val


def feature_match_index(feat_input, feat_ref, patch_size=3, input_stride=1, ref_stride=1, is_norm=True,
                        norm_input=False):
    """Drop-in for mmsr/models/archs/ref_map_util.py:26-86 (same signature, same return)."""
    idx, val = corr_argmax(feat_input.unsqueeze(0), feat_ref.unsqueeze(0), patch_size, input_stride, ref_stride,
                           is_norm, norm_input)
    return idx[0], val[0]


def offset_pyramid(idx, scale, ref_gw=None):
    """idx int64 [B,gh,gw] -> pre_offset [B,9,s*(gh+2),s*(gw+2),2] (x,y)."""
    _require_cuda('idx', idx, torch.int64)
    idx = idx.contiguous()
    B, gh, gw = idx.shape
    out = torch.empty(B, 9, scale * (gh + 2), scale * (gw + 2), 2, dtype=torch.float32, device=idx.device)
    _call('c2m_offset_pyramid_f32', idx, B, gh, gw, ref_gw or gw, scale, out, device=idx.device)
    return out


def _dense_nchw_or_nhwc(t):
    """Accept NCHW-contiguous or channels-last storage without copying; otherwise make NCHW."""
    if t.is_contiguous() or t.is_contiguous(memory_format=torch.channels_last):
        return t
    return t.contiguous()


def _shape(x, cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, out):
    s = DcnShape()
    s.B, s.C, s.H, s.W = x.shape
    s.Cout = cout
    s.kh, s.kw, s.sh, s.sw, s.ph, s.pw, s.dh, s.dw, s.dg = kh, kw, sh, sw, ph, pw, dh, dw, dg
    s.xs_b, s.xs_c, s.xs_y, s.xs_x = x.stride()
    s.os_b, s.os_c, s.os_y, s.os_x = out.stride()
    return s


def _out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw):
    return ((H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1)


def _deform_out(x, weight, offset, mask, geom, deformable_group, grad_output=None, nonempty=False):
    """(Ho, Wo) of the deformable convolution of x [B, C, H, W] by weight [Cout, ...] with geom = (kh, kw, sh, sw, ph,
    pw, dh, dw).  Refuses, in this order: an empty output (when nonempty), a grad_output (when given) that is not
    [B, Cout, Ho, Wo], an offset that is not [B, 2*dg*kh*kw, Ho, Wo] or a mask (when given) that is not
    [B, dg*kh*kw, Ho, Wo]."""
    B, _, H, W = x.shape
    Ho, Wo = _out_hw(H, W, *geom)
    if nonempty and (Ho < 1 or Wo < 1):
        raise RuntimeError(f'convolution input is too small (output would be {Ho} x {Wo})')
    want = (B, weight.shape[0], Ho, Wo)
    if grad_output is not None and tuple(grad_output.shape) != want:
        raise RuntimeError(f'grad_output has shape {tuple(grad_output.shape)}, expected {want}')
    T = geom[0] * geom[1]
    if tuple(offset.shape) != (B, 2 * deformable_group * T, Ho, Wo) or (
            mask is not None and tuple(mask.shape) != (B, deformable_group * T, Ho, Wo)):
        raise RuntimeError(f'offset/mask shape mismatch: {tuple(offset.shape)}, '
                           f'{None if mask is None else tuple(mask.shape)} for output {Ho}x{Wo}')
    return Ho, Wo


def _pre_offset_source(pre_offset, idx, B, taps, Ho, Wo):
    """Checks the optional pre-offset source of the fused DCN forwards and returns (pre_offset, idx), each
    contiguous or None: pre_offset [B,taps,Ho,Wo,2] (x,y) fp32 wins over idx int64 [B,gh,gw]."""
    if pre_offset is not None:
        _require_cuda('pre_offset', pre_offset)
        if tuple(pre_offset.shape) != (B, taps, Ho, Wo, 2):
            raise RuntimeError(f'pre_offset has shape {tuple(pre_offset.shape)}')
        return pre_offset.contiguous(), None
    if idx is not None:
        _require_cuda('idx', idx, torch.int64)
        return None, idx.contiguous()
    return None, None


def dcn_v2_forward(input, weight, bias, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                   dilation_h, dilation_w, deformable_group):
    """`_ext.dcn_v2_forward` (DCNv2/src/dcn_v2.h:9-39; call site dcn_v2.py:26-30)."""
    for n, t in (('input', input), ('weight', weight), ('bias', bias), ('offset', offset), ('mask', mask)):
        _require_cuda(n, t)
    if weight.shape[2] != kernel_h or weight.shape[3] != kernel_w:
        raise RuntimeError(f'Input shape and kernel shape wont match: ({kernel_h} x {kernel_w} vs '
                           f'{weight.shape[2]} x {weight.shape[3]}).')
    if input.shape[1] != weight.shape[1]:
        raise RuntimeError(f'Input shape and kernel channels wont match: ({input.shape[1]} vs {weight.shape[1]}).')
    geom = (kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w)
    x = _dense_nchw_or_nhwc(input)
    Ho, Wo = _deform_out(x, weight, offset, mask, geom, deformable_group)
    if (geom == (3, 3, 1, 1, 1, 1, 1, 1) and dcn_tc_supported(x.shape[1], weight.shape[0], deformable_group) and
            os.environ.get('C2M_EXT_DCN_TC', '1') != '0'):
        # eligible shapes (every DCN of C2-Matching) take the tensor-core kernel: fp32 NCHW -> packed-split operand
        # in one pass, final offsets / mask read as given, fp32 NCHW out.  The FFMA kernel below stays the general
        # path (any kernel size / stride / dilation / group width).
        return dcn_v2_fused_tc(x, offset.contiguous(), weight, bias, deformable_group, final_mask=mask.contiguous())
    return _deform_forward(x, weight, offset, mask, bias, Ho, Wo, geom, 1, deformable_group)


def dcn_v2_fused_forward(x, om, weight, bias, deformable_group, pre_offset=None, idx=None, pre_scale=1,
                         ref_gw=None, lrelu_slope=1.0, channels_last_out=False):
    """Tail of DCN_sep_pre_multi_offset.forward (dcn_v2.py:229-253) in one kernel: `om` is the raw
    conv_offset_mask output.  Either `pre_offset` [B,9,H,W,2] or `idx` [B,gh,gw] (+pre_scale)."""
    _require_cuda('x', x)
    _require_cuda('om', om)
    x = _dense_nchw_or_nhwc(x)
    om = om.contiguous()
    B, C, H, W = x.shape
    kh, kw = weight.shape[2:]
    Ho, Wo = _out_hw(H, W, kh, kw, 1, 1, kh // 2, kw // 2, 1, 1)
    if tuple(om.shape) != (B, 3 * deformable_group * kh * kw, Ho, Wo):
        raise RuntimeError(f'conv_offset_mask output has shape {tuple(om.shape)}')
    out = _empty_f32(B, weight.shape[0], Ho, Wo, x.device, channels_last_out)
    s = _shape(x, weight.shape[0], kh, kw, 1, 1, kh // 2, kw // 2, 1, 1, deformable_group, out)
    pre_offset, idx = _pre_offset_source(pre_offset, idx, B, kh * kw, Ho, Wo)
    gh, gw = idx.shape[1:] if idx is not None else (0, 0)
    _call('c2m_dcn_v2_fused_forward_f32', x, om, pre_offset, idx, gh, gw, ref_gw or gw, pre_scale, weight.contiguous(),
          bias.contiguous() if bias is not None else None, float(lrelu_slope), out, s, device=x.device)
    return out


# ------------------------------------------------------------------------------------------------
# Packed-split activations ("PSA") and the tensor-core 3x3 convolution (include/c2m_sm100.h)
class PSA:
    """fp16 hi/lo planes [B][ceil(C/8)][H][W][8]; value = (hi + lo) * 2^-sa."""
    __slots__ = ('hi', 'lo', 'B', 'C', 'H', 'W', 'sa')

    def __init__(self, hi, lo, B, C, H, W, sa=0):
        self.hi, self.lo, self.B, self.C, self.H, self.W, self.sa = hi, lo, B, C, H, W, sa

    @staticmethod
    def empty(B, C, H, W, device, sa=0):
        c8 = (C + 7) // 8
        buf = torch.empty(2, B, c8, H, W, 8, dtype=torch.float16, device=device)
        return PSA(buf[0], buf[1], B, C, H, W, sa)

    @property
    def shape(self):
        return (self.B, self.C, self.H, self.W)


class OctF32:
    """fp32 tensor in the octet-planar layout [B][ceil(C/8)][H][W][8] (padding channels are 0): what
    conv3x3_psa(..., f32_octets=True) writes with two 16 B stores per octet and what the tensor-core DCN reads
    its offsets / mask from.  `.nchw()` gives the ordinary [B,C,H,W] tensor."""
    __slots__ = ('data', 'C')

    def __init__(self, data, C):
        self.data, self.C = data, C

    @property
    def shape(self):
        B, _, H, W, _ = self.data.shape
        return (B, self.C, H, W)

    def nchw(self):
        B, c8, H, W, _ = self.data.shape
        return self.data.permute(0, 1, 4, 2, 3).reshape(B, c8 * 8, H, W)[:, :self.C].contiguous()


def suggest_sa(amax, target_log2=12):
    """Scale exponent for a PSA tensor whose largest magnitude is `amax`: amax * 2^sa ~ 2^target_log2 (fp16 tops out
    at 65504 = 2^16, so 16x headroom; values below 2^-14 * 2^-sa lose their lo half to fp16 subnormals)."""
    if not (amax > 0) or not math.isfinite(amax):
        return 0
    return max(-14, min(24, target_log2 - math.ceil(math.log2(amax))))


def psa_amax(p):
    """Largest |value| of a PSA tensor (from its hi half: within 2^-11), as a Python float (synchronises)."""
    return float(p.hi.abs().max()) * 2.0 ** (-p.sa)


def psa_from_f32(x, sa=0):
    _require_cuda('x', x)
    B, C, H, W = x.shape
    out = PSA.empty(B, C, H, W, x.device, sa)
    _call('c2m_psa_from_f32', x, B, C, H, W, *x.stride(), sa, out.hi, out.lo, device=x.device)
    return out


def _strided_like(add, out, channels_last):
    """`add` with the shape and strides of `out` (copied into the layout `channels_last` names when they differ)."""
    if add.shape != out.shape or add.stride() != out.stride():
        return add.contiguous(memory_format=_memory_format(channels_last))
    return add


def psa_to_f32(p, add=None, channels_last=False):
    out = _empty_f32(p.B, p.C, p.H, p.W, p.hi.device, channels_last)
    if add is not None:
        _require_cuda('add', add)
        add = _strided_like(add, out, channels_last)
    _call('c2m_psa_to_f32', p.hi, p.lo, p.B, p.C, p.H, p.W, p.sa, add, out, *out.stride(), device=out.device)
    return out


def psa_maxpool2(p):
    """nn.MaxPool2d(kernel_size=2, stride=2) on a PSA tensor."""
    out = PSA.empty(p.B, p.C, p.H // 2, p.W // 2, p.hi.device, p.sa)
    _call('c2m_psa_maxpool2', p.hi, p.lo, p.B, p.C, p.H, p.W, out.hi, out.lo, device=p.hi.device)
    return out


def conv3x3_supported(H, W):
    """The tensor-core kernel takes any channel counts; maps must hold one halo tile (18 x 10)."""
    return H >= 18 and W >= 10


# ---- packed-weight cache.  The blob lives ON the tensor object (so it dies with it — a global cache keyed
# by data_ptr would alias a freed parameter's address) and is re-made when the storage, the shape or the
# version counter changes.  Writes through `.data` do NOT bump the version: call invalidate_packs() after
# such an edit (load_state_dict / `with torch.no_grad(): p.copy_()` do bump it).
_fallback_packs = {}          # id(tensor) -> (weakref, {attr: entry}) for tensors that refuse attributes
_PACK_ATTRS = ('_c2m_pack', '_c2m_pack_dgrad', '_c2m_dcn_pack', '_c2m_dcn_pack_dgrad')


def _pack_cached(weight, attr, extra, size_fn, pack_fn, dims, source=None):
    """The blob of `weight` cached under `attr` (one of _PACK_ATTRS), packed on a miss: size_fn(*dims) bytes filled by
    pack_fn(w, *dims, blob, stream), where w is source(weight) (default: the weight itself) made contiguous.  `extra`
    is part of the cache key."""
    tag = (weight.data_ptr(), weight._version, tuple(weight.shape), extra)
    store = getattr(weight, '__dict__', None)
    if store is None:
        ent = _fallback_packs.get(id(weight))
        if ent is None or ent[0]() is not weight:
            key = id(weight)
            ent = (weakref.ref(weight, lambda _r, key=key: _fallback_packs.pop(key, None)), {})
            _fallback_packs[key] = ent
        store = ent[1]
    cached = store.get(attr)
    cur = torch.cuda.current_stream(weight.device)
    if cached is not None and cached[0] == tag:
        _, blob, ev, st = cached
        if st != cur.cuda_stream and not torch.cuda.is_current_stream_capturing():
            # packed on another stream: order this stream after the pack kernels.  (A capturing stream cannot wait on
            # an event recorded outside its capture; RestorationPipeline synchronises the device before it captures.)
            cur.wait_event(ev)
        return blob
    w = weight.detach()
    w = (source(w) if source else w).contiguous()
    # unsupported dims size to 0 without an error message; the pack call then reports them
    blob = torch.empty(getattr(_lib.lib(), size_fn)(*dims), dtype=torch.uint8, device=weight.device)
    _call(pack_fn, w, *dims, blob, device=weight.device)
    ev = torch.cuda.Event()
    ev.record(cur)
    store[attr] = (tag, blob, ev, cur.cuda_stream)
    return blob


def invalidate_packs(obj):
    """Drop the cached packed weights of a tensor, or of every parameter of a module (needed after in-place
    edits through `.data`, which do not bump the tensor version)."""
    tensors = [obj] if isinstance(obj, torch.Tensor) else list(obj.parameters())
    if not isinstance(obj, torch.Tensor):
        for m in obj.modules():                 # calibrated PSA scale exponents of VGG trunks depend on the weights too
            m.__dict__.pop('_c2m_sa', None)
    for t in tensors:
        d = getattr(t, '__dict__', None)
        if d is not None:
            for attr in _PACK_ATTRS:
                d.pop(attr, None)
        _fallback_packs.pop(id(t), None)


def conv3x3_pack_weights(weight, dgrad=False):
    """Pack a [Cout,Cin,3,3] fp32 weight for c2m_conv3x3_psa (cached, see _pack_cached).  dgrad: pack the weights of the
    input gradient instead, W'[ci][co][ky][kx] = W[co][ci][2-ky][2-kx] (a Cout -> Cin convolution)."""
    _require_cuda('weight', weight)
    cout, cin = weight.shape[:2]
    if dgrad:
        return _pack_cached(weight, '_c2m_pack_dgrad', None, 'c2m_conv3x3_packed_weight_bytes',
                            'c2m_conv3x3_pack_weights_f32', (cout, cin), lambda w: w.transpose(0, 1).flip(2, 3))
    return _pack_cached(weight, '_c2m_pack', None, 'c2m_conv3x3_packed_weight_bytes', 'c2m_conv3x3_pack_weights_f32',
                        (cin, cout))


_ACT = {None: 0, 'none': 0, 'relu': 1, 'lrelu': 2}


def conv3x3_psa(x, weight, bias, act=None, residual=None, residual2=None, x2=None, out=None, sa_out=0,
                pixel_shuffle=0, out_f32=False, add_f32=None, psa_out=True, channels_last=False, f32_octets=False,
                packed=None, x_amax=None):
    """y = act(conv3x3(cat[x, x2], weight) + bias), fp32-grade on tensor cores.
    f32_octets: the fp32 result is an OctF32 (octet-planar) instead of a strided tensor.
    packed: a packed blob of `weight` made elsewhere (the input gradient's rotated weights); `weight` then only gives
    the shape.
    x_amax: the per-image amax of `x` from _conv3x3_operand (x.sa is then unused).

    Returns the PSA tensor `y + residual + residual2` (or PixelShuffle(2)(y)), and/or — with
    out_f32=True — the fp32 tensor `y + add_f32`.  With both, returns (psa, f32)."""
    cout, cin = weight.shape[:2]
    c_in = x.C + (x2.C if x2 is not None else 0)
    if cin != c_in:
        raise RuntimeError(f'conv3x3_psa: weight expects {cin} input channels, got {c_in}')
    blob = conv3x3_pack_weights(weight) if packed is None else packed
    dev = x.hi.device
    a = _lib.ConvArgs()
    a.in_hi, a.in_lo, a.Cin = x.hi.data_ptr(), x.lo.data_ptr(), x.C
    if x2 is not None:
        if (x2.B, x2.H, x2.W) != (x.B, x.H, x.W) or x2.sa != x.sa:
            raise RuntimeError('conv3x3_psa: concatenated inputs must share batch / size / scale')
        a.in2_hi, a.in2_lo, a.Cin2 = x2.hi.data_ptr(), x2.lo.data_ptr(), x2.C
    a.B, a.H, a.W, a.sa_in = x.B, x.H, x.W, x.sa
    a.x_amax = _ptr(x_amax)
    a.packed_w, a.bias = blob.data_ptr(), _ptr(bias)
    a.Cout, a.act = cout, _ACT[act]
    for r, (fh, fl) in ((residual, ('res_hi', 'res_lo')), (residual2, ('res2_hi', 'res2_lo'))):
        if r is not None:
            if r.shape != (x.B, cout, x.H, x.W):
                raise RuntimeError(f'conv3x3_psa: residual shape {r.shape}')
            setattr(a, fh, r.hi.data_ptr())
            setattr(a, fl, r.lo.data_ptr())
            a.sa_res = r.sa
    a.pixel_shuffle = pixel_shuffle
    ret_psa = None
    if psa_out:
        if out is None:
            if pixel_shuffle == 2:
                out = PSA.empty(x.B, cout // 4, 2 * x.H, 2 * x.W, dev, sa_out)
            else:
                out = PSA.empty(x.B, cout, x.H, x.W, dev, sa_out)
        a.out_hi, a.out_lo, a.sa_out = out.hi.data_ptr(), out.lo.data_ptr(), out.sa
        ret_psa = out
    ret_f32 = None
    if out_f32 and f32_octets:
        if add_f32 is not None:
            raise RuntimeError('conv3x3_psa: add_f32 is not available with f32_octets')
        ret_f32 = OctF32(torch.empty(x.B, (cout + 7) // 8, x.H, x.W, 8, dtype=torch.float32, device=dev), cout)
        a.out_f32, a.out_f32_octets = ret_f32.data.data_ptr(), 1
    elif out_f32:
        ret_f32 = _empty_f32(x.B, cout, x.H, x.W, dev, channels_last)
        a.out_f32 = ret_f32.data_ptr()
        a.os_b, a.os_c, a.os_y, a.os_x = ret_f32.stride()
        if add_f32 is not None:
            add_f32 = _strided_like(add_f32, ret_f32, channels_last)
            a.add_f32 = add_f32.data_ptr()
    _call('c2m_conv3x3', ctypes.addressof(a), device=dev)
    return _one_or_both(ret_psa, ret_f32)


def _conv3x3_operand(x):
    """x [B,C,H,W] fp32 (any strides, any magnitude) as PSA image b times 2^sa_b, and the [B] amax buffer the kernels
    read sa_b from (c2m_conv3x3_operand_f32).  The operand form of x in the convolution's forward and of grad_output in
    both backwards.  Call with x's device current."""
    B, C, H, W = x.shape
    xp = PSA.empty(B, C, H, W, x.device)
    amax = torch.empty(B, dtype=torch.int32, device=x.device)
    _call('c2m_conv3x3_operand_f32', x, B, C, H, W, *x.stride(), xp.hi, xp.lo, amax)
    return xp, amax


class _Conv3x3(torch.autograd.Function):
    """Forward on conv3x3_wgmma_kernel from x at a power-of-two scale per image chosen on the device
    (c2m_conv3x3_operand_f32); backward: the activation's backward, dX on the same kernel with the rotated weights, dW
    on conv3x3_wgrad_kernel, db as a torch sum.  grad_output enters the kernels like x, as PSA at a power-of-two scale
    per image chosen on the device.  The results divide every scale back out on the device, image by image."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        with torch.cuda.device(x.device):
            xp, x_amax = _conv3x3_operand(x)
        y = conv3x3_psa(xp, weight, bias, act=act, psa_out=False, out_f32=True, x_amax=x_amax)
        ctx.act = act
        ctx.save_for_backward(xp.hi, xp.lo, x_amax, weight, y if act else None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x_hi, x_lo, x_amax, weight, y = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        B, c8, H, W, _ = x_hi.shape
        cout, cin = weight.shape[:2]
        if ctx.act == 'relu':
            gy = torch.where(y > 0, gy, 0.)
        elif ctx.act == 'lrelu':
            gy = torch.where(y > 0, gy, gy * 0.1)
        dev = gy.device
        dx = dw = db = None
        with torch.cuda.device(dev):
            gp, amax = _conv3x3_operand(gy)
            if need_x:
                dx = conv3x3_psa(gp, weight.transpose(0, 1), None, psa_out=False, out_f32=True,
                                 packed=conv3x3_pack_weights(weight, dgrad=True), x_amax=amax)
            if need_w:
                dw = torch.empty(cout, cin, 3, 3, dtype=torch.float32, device=dev)
                nbytes = _size('c2m_conv3x3_wgrad_workspace_bytes', B, cin, cout, H, W)
                ws = _workspace(nbytes, dev)
                _call('c2m_conv3x3_wgrad_scaled', gp.hi, gp.lo, amax, x_hi, x_lo, x_amax, B, cin, cout, H, W, dw, ws,
                      nbytes)
            if need_b:
                db = gy.sum((0, 2, 3))
        return dx, dw, db, None


def conv3x3(x, weight, bias=None, act=None):
    """Differentiable act(conv2d(x, weight, bias, stride 1, padding 1)) on the tensor cores, fp32-grade forward and
    backward (fp32 in, fp32 out).  x [B,Cin,H,W] with H >= 18 and W >= 10, weight [Cout,Cin,3,3], bias [Cout] or None,
    act None / 'relu' / 'lrelu' (LeakyReLU(0.1)).  Any fp32 magnitude: each image of x and grad_output enters the
    kernels at its own power-of-two scale chosen on the device from its largest finite value, so an image's results do
    not depend on the other images' magnitudes, x * 2^k gives exactly 2^k times the output and dW, and grad_output * 2^k
    exactly 2^k times every gradient.  NaN / Inf propagate to the entries that depend on them, as in an fp32 convolution (the
    input gradient of a non-finite weight also reaches the map's border)."""
    _require_cuda('x', x)
    _require_cuda('weight', weight)
    if bias is not None:
        _require_cuda('bias', bias)
    if act not in (None, 'relu', 'lrelu'):
        raise ValueError(f'conv3x3: act must be None, relu or lrelu, got {act!r}')
    if x.dim() != 4 or weight.dim() != 4 or tuple(weight.shape[1:]) != (x.shape[1], 3, 3):
        raise RuntimeError(f'conv3x3: weight {tuple(weight.shape)} does not fit input {tuple(x.shape)} '
                           '(expected [Cout, Cin, 3, 3])')
    if bias is not None and tuple(bias.shape) != (weight.shape[0],):
        raise RuntimeError(f'conv3x3: bias {tuple(bias.shape)} does not fit {weight.shape[0]} output channels')
    if not conv3x3_supported(x.shape[2], x.shape[3]):
        raise RuntimeError(f'conv3x3: map {x.shape[2]}x{x.shape[3]} smaller than one halo tile (18x10)')
    return _Conv3x3.apply(x, weight, bias, act)


# ------------------------------------------------------------------------------------------------
# DCNv2 on tensor cores
def dcn_tc_supported(C, Cout, dg, kh=3, kw=3):
    return kh == 3 and kw == 3 and bool(_lib.lib().c2m_dcn_tc_supported(C, Cout, dg))


def _dcn_tc_pack(weight, dg):
    cout, c = weight.shape[:2]
    return _pack_cached(weight, '_c2m_dcn_pack', dg, 'c2m_dcn_tc_packed_weight_bytes', 'c2m_dcn_tc_pack_weights_f32',
                        (c, cout, dg))


def _dcn_tc_operand(x, dg, mask=None):
    """The tensor-core DCN's interleaved operand x_il of x, with its x_amax and mask_amax buffers.  x is a PSA tensor at
    scale exponent 0 (both buffers None) or fp32 [B,C,H,W], dense NCHW or channels-last, of any magnitude: x_il then
    holds image b times 2^sa_b, x_amax its [B] exponents and, given the final mask [B,dg*9,H,W], mask_amax the mask's
    (else None), all taken on the device.  Call with x's device current."""
    B, C, H, W = x.shape
    dev = x.hi.device if isinstance(x, PSA) else x.device
    x_il = torch.empty(_lib.lib().c2m_dcn_tc_operand_bytes(B, C, H, W, dg) // 2, dtype=torch.float16, device=dev)
    if isinstance(x, PSA):
        _call('c2m_dcn_tc_operand_psa', x.hi, x.lo, B, C, H, W, dg, x_il)
        return x_il, None, None
    amax = torch.empty(2 * B, dtype=torch.int32, device=dev)
    _call('c2m_dcn_tc_operand_f32', x, B, C, H, W, *x.stride(), dg, mask, x_il, amax)
    return x_il, amax[:B], None if mask is None else amax[B:]


def dcn_v2_fused_tc(x, om, weight, bias, deformable_group, pre_offset=None, idx=None, pre_scale=1, ref_gw=None,
                    lrelu=False, psa_out=False, out_f32=True, channels_last_out=False, final_mask=None):
    """Tensor-core version of dcn_v2_fused_forward (3x3/s1/p1/d1).  Returns fp32 and / or PSA.
    final_mask: `om` then holds the FINAL offsets [B,2*dg*9,H,W] and final_mask the FINAL modulation
    [B,dg*9,H,W] (the `_ext.dcn_v2_forward` contract: no pre-offsets, no sigmoid)."""
    om_oct = isinstance(om, OctF32)
    _require_cuda('om', om.data if om_oct else om)
    xp = x if isinstance(x, PSA) else getattr(x, '_c2m_psa', None)
    if xp is not None and xp.shape != tuple(x.shape):
        xp = None
    if xp is not None:
        if xp.sa != 0:
            raise RuntimeError('dcn_v2_fused_tc: PSA input must have scale exponent 0')
        x, dev = xp, xp.hi.device
    else:
        _require_cuda('x', x)
        x = _dense_nchw_or_nhwc(x)
        dev = x.device
    B, C, H, W = x.shape
    cout = weight.shape[0]
    if final_mask is not None:
        _require_cuda('final_mask', final_mask)
        if om_oct or pre_offset is not None or idx is not None:
            raise RuntimeError('dcn_v2_fused_tc: final_mask excludes octet-planar om and pre-offsets')
        if tuple(om.shape) != (B, 18 * deformable_group, H, W) or tuple(final_mask.shape) != (B, 9 * deformable_group, H, W):
            raise RuntimeError(f'offset/mask shape mismatch: {tuple(om.shape)}, {tuple(final_mask.shape)}')
    elif tuple(om.shape) != (B, 27 * deformable_group, H, W):
        raise RuntimeError(f'conv_offset_mask output has shape {tuple(om.shape)}')
    if final_mask is not None:
        final_mask = final_mask.contiguous()
    a = _lib.DcnTcArgs()
    # every tensor whose address `a` holds stays referenced here until the launch below is enqueued (same stream)
    with torch.cuda.device(dev):
        x_il, x_amax, mask_amax = _dcn_tc_operand(x, deformable_group, final_mask)
        a.x_il, a.x_amax, a.mask_amax, a.mask = x_il.data_ptr(), _ptr(x_amax), _ptr(mask_amax), _ptr(final_mask)
        if om_oct:
            a.om, a.om_octets = om.data.data_ptr(), 1
        else:
            om = om.contiguous()
            a.om = om.data_ptr()
        pre_offset, idx = _pre_offset_source(pre_offset, idx, B, 9, H, W)
        if pre_offset is not None:
            a.pre = pre_offset.data_ptr()
        elif idx is not None:
            a.idx = idx.data_ptr()
            a.gh, a.gw = idx.shape[1:]
            a.ref_gw, a.pre_scale = (ref_gw or idx.shape[2]), pre_scale
        a.B, a.C, a.H, a.W, a.Cout, a.dg = B, C, H, W, cout, deformable_group
        blob = _dcn_tc_pack(weight, deformable_group)
        a.packed_w = blob.data_ptr()
        bias = bias.contiguous() if bias is not None else None
        a.bias = _ptr(bias)
        a.lrelu = int(bool(lrelu))
        ret_p = ret_f = None
        if psa_out:
            ret_p = PSA.empty(B, cout, H, W, dev)
            a.out_hi, a.out_lo, a.sa_out = ret_p.hi.data_ptr(), ret_p.lo.data_ptr(), 0
        if out_f32:
            ret_f = _empty_f32(B, cout, H, W, dev, channels_last_out)
            a.out_f32 = ret_f.data_ptr()
            a.os_b, a.os_c, a.os_y, a.os_x = ret_f.stride()
        _call('c2m_dcn_v2_fused_tc', ctypes.addressof(a))
    return _one_or_both(ret_p, ret_f)


def _dcn_tc_pack_dgrad(weight, dg):
    cout, c = weight.shape[:2]
    return _pack_cached(weight, '_c2m_dcn_pack_dgrad', dg, 'c2m_dcn_tc_dgrad_packed_weight_bytes',
                        'c2m_dcn_tc_pack_dgrad_weights_f32', (c, cout, dg))


class _DcnV2Tc(torch.autograd.Function):
    """Forward: the tensor-core launch of `_ext.dcn_v2_forward` (dcn_v2_fused_tc with the final mask).  Backward:
    grad_output as PSA at a power-of-two scale per image chosen on the device (c2m_conv3x3_operand_f32), then
    dcn_dgrad_kernel for grad_offset / grad_mask (and grad_input when x requires it) and dcn_wgrad_kernel for the
    weight gradient; db is a torch sum.  Every gradient divides each image's scales back out, so an image's gradients
    do not depend on the other images' magnitudes."""

    @staticmethod
    def forward(ctx, x, offset, mask, weight, bias, dg):
        offset, mask = offset.contiguous(), mask.contiguous()
        ctx.dg = dg
        ctx.save_for_backward(x, offset, mask, weight)
        return dcn_v2_fused_tc(x, offset, weight, bias, dg, final_mask=mask)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy):
        x, offset, mask, weight = ctx.saved_tensors
        need_x, need_off, need_mask, need_w, need_b = ctx.needs_input_grad[:5]
        dg = ctx.dg
        x = _dense_nchw_or_nhwc(x)
        B, C, H, W = x.shape
        cout = weight.shape[0]
        gy = gy.contiguous()
        dev = gy.device
        gx = goff = gmask = dw = db = None
        with torch.cuda.device(dev):
            gp, gamax = _conv3x3_operand(gy)
            # the forward's operand, made again: x * 2^sa and mask * 2^sm per image
            x_il, x_amax, mask_amax = _dcn_tc_operand(x, dg, mask)
            a = _lib.DcnTcGradArgs()
            a.gy_hi, a.gy_lo, a.gy_amax = gp.hi.data_ptr(), gp.lo.data_ptr(), gamax.data_ptr()
            a.x_il, a.x_amax, a.mask_amax = x_il.data_ptr(), x_amax.data_ptr(), mask_amax.data_ptr()
            a.offset, a.mask = offset.data_ptr(), mask.data_ptr()
            a.B, a.C, a.H, a.W, a.Cout, a.dg = B, C, H, W, cout, dg
            if need_x or need_off or need_mask:
                goff, gmask = torch.empty_like(offset), torch.empty_like(mask)
                a.packed_w = _dcn_tc_pack_dgrad(weight, dg).data_ptr()
                a.grad_offset, a.grad_mask = goff.data_ptr(), gmask.data_ptr()
                if need_x:
                    gx = torch.zeros(B, C, H, W, dtype=torch.float32, device=dev)
                    a.grad_input = gx.data_ptr()
                _call('c2m_dcn_tc_dgrad', ctypes.addressof(a))
            if need_w:
                dw = torch.empty(cout, C, 3, 3, dtype=torch.float32, device=dev)
                nbytes = _size('c2m_dcn_tc_wgrad_workspace_bytes', B, C, H, W, cout, dg)
                ws = _workspace(nbytes, dev)
                a.grad_weight, a.ws, a.ws_bytes = dw.data_ptr(), ws.data_ptr(), nbytes
                _call('c2m_dcn_tc_wgrad', ctypes.addressof(a))
            if need_b:
                db = gy.sum((0, 2, 3))
        return (gx, goff if need_off else None, gmask if need_mask else None, dw, db, None)


def dcn_tc_backward_supported(C, Cout, dg, H, W):
    """Shapes the tensor-core DCN backward takes: the forward's (dcn_tc_supported) on maps of at least 16 x 8."""
    return dcn_tc_supported(C, Cout, dg) and H >= 16 and W >= 8


def dcn_v2_tc(x, offset, mask, weight, bias, deformable_group):
    """Differentiable modulated deformable convolution, 3x3 / stride 1 / pad 1 / dilation 1, on the tensor cores
    forward and backward (fp32-grade).  The `_ext` contract: final offsets [B,2*dg*9,H,W] and final mask [B,dg*9,H,W];
    the output equals `_ext.dcn_v2_forward`'s tensor-core route bit for bit.  Gradients flow to every input that
    requires one; grad_input is summed with atomics, every other gradient in a fixed order."""
    for n, t in (('x', x), ('offset', offset), ('mask', mask), ('weight', weight)):
        _require_cuda(n, t)
    if bias is not None:
        _require_cuda('bias', bias)
    B, C, H, W = x.shape
    if tuple(weight.shape) != (weight.shape[0], C, 3, 3):
        raise RuntimeError(f'dcn_v2_tc: weight {tuple(weight.shape)} does not fit input {tuple(x.shape)}')
    if not dcn_tc_backward_supported(C, weight.shape[0], deformable_group, H, W):
        raise RuntimeError(f'dcn_v2_tc: C={C} Cout={weight.shape[0]} dg={deformable_group} on {H}x{W} unsupported')
    return _DcnV2Tc.apply(x, offset, mask, weight, bias, deformable_group)


# ------------------------------------------------------------------------------------------------
# DCNv2 backward (training; completes the `_ext` ABI)
def dcn_v2_backward(input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                    pad_w, dilation_h, dilation_w, deformable_group):
    """`_ext.dcn_v2_backward` (DCNv2/src/dcn_v2.h:41-72; call site dcn_v2.py:38-47) ->
    [grad_input, grad_offset, grad_mask, grad_weight, grad_bias]: the groups = 1 case of deform_conv_backward,
    behind `_ext`'s own checks."""
    for n, t in (('input', input), ('weight', weight), ('bias', bias), ('offset', offset), ('mask', mask),
                 ('grad_output', grad_output)):
        _require_cuda(n, t)
    x, w = input.contiguous(), weight.contiguous()
    offset, mask, gout = offset.contiguous(), mask.contiguous(), grad_output.contiguous()
    geom = (kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w)
    _deform_out(x, w, offset, mask, geom, deformable_group, grad_output=gout)
    s = _shape(x, w.shape[0], *geom, deformable_group, gout)
    return list(_deform_backward(x, w, offset, mask, gout, s, 1, True, True))


# ------------------------------------------------------------------------------------------------
# Deformable PS-ROI pooling (completes the `_ext` ABI)
def _psroi_prepare(input, bbox, trans, no_trans, spatial_scale, output_dim, group_size, pooled_size, part_size,
                   sample_per_part, trans_std):
    """Validates the tensors (the size / channel rules are checked again by the library) and returns the contiguous
    operands and the c2m_psroi_shape."""
    if not isinstance(input, torch.Tensor):
        raise TypeError('input must be a Tensor')
    dtype = input.dtype
    if dtype not in (torch.float32, torch.float64):
        raise RuntimeError(f'input must be torch.float32 or torch.float64, got {dtype}')
    _require_cuda('input', input, dtype)
    _require_cuda('bbox', bbox, dtype)
    if not no_trans:
        _require_cuda('trans', trans, dtype)
    if input.dim() != 4:
        raise RuntimeError(f'input must be [B, C, H, W], got shape {tuple(input.shape)}')
    if bbox.dim() != 2 or bbox.shape[1] != 5:
        raise RuntimeError(f'bbox must be [R, 5], got shape {tuple(bbox.shape)}')
    if bbox.device != input.device or (not no_trans and trans.device != input.device):
        raise RuntimeError('input, bbox and trans must be on the same device')
    if min(pooled_size, part_size, sample_per_part) < 1:
        raise RuntimeError(f'pooled_size, part_size and sample_per_part must be >= 1, got {pooled_size}, '
                           f'{part_size}, {sample_per_part}')
    B, C, H, W = input.shape
    R = bbox.shape[0]
    K = 1
    if not no_trans:
        if (trans.dim() != 4 or trans.shape[0] != R or trans.shape[1] < 2 or trans.shape[1] % 2 or
                tuple(trans.shape[2:]) != (part_size, part_size)):
            raise RuntimeError(f'trans must be [R, 2K, part_size, part_size] = [{R}, 2K, {part_size}, {part_size}] '
                               f'with K >= 1, got shape {tuple(trans.shape)}')
        K = trans.shape[1] // 2
    s = _lib.PsroiShape(B=B, C=C, H=H, W=W, R=R, no_trans=int(bool(no_trans)), num_classes=K,
                        spatial_scale=spatial_scale, trans_std=trans_std, output_dim=output_dim,
                        group_size=group_size, pooled_size=pooled_size, part_size=part_size,
                        sample_per_part=sample_per_part)
    return s, input.contiguous(), bbox.contiguous(), None if no_trans else trans.contiguous()


def dcn_v2_psroi_pooling_forward(input, bbox, trans, no_trans, spatial_scale, output_dim, group_size, pooled_size,
                                 part_size, sample_per_part, trans_std):
    """`_ext.dcn_v2_psroi_pooling_forward` (DCNv2/src/dcn_v2.h:75-108; call site dcn_v2.py:280-283) ->
    (output, output_count), both [R, output_dim, pooled_size, pooled_size] in the input's dtype."""
    s, x, bbox, trans = _psroi_prepare(input, bbox, trans, no_trans, spatial_scale, output_dim, group_size,
                                       pooled_size, part_size, sample_per_part, trans_std)
    out = torch.empty(s.R, output_dim, pooled_size, pooled_size, dtype=x.dtype, device=x.device)
    count = torch.empty_like(out)
    _call(f'c2m_psroi_pooling_forward_{_DTYPE_SFX[x.dtype]}', x, bbox, trans, s, out, count, device=x.device)
    return out, count


def dcn_v2_psroi_pooling_backward(out_grad, input, bbox, trans, top_count, no_trans, spatial_scale, output_dim,
                                  group_size, pooled_size, part_size, sample_per_part, trans_std):
    """`_ext.dcn_v2_psroi_pooling_backward` (DCNv2/src/dcn_v2.h:110-144; call site dcn_v2.py:291-304) ->
    (grad_input, grad_trans).  grad_input is scattered with atomics (summation order not fixed), or, when torch's
    deterministic algorithms are enabled, gathered in a fixed order; grad_trans is reduced in a fixed order and is the
    same bit for bit on every run.  With no_trans, grad_trans is
    zeros_like(trans)."""
    s, x, bbox, tr = _psroi_prepare(input, bbox, trans, no_trans, spatial_scale, output_dim, group_size, pooled_size,
                                    part_size, sample_per_part, trans_std)
    _require_cuda('out_grad', out_grad, x.dtype)
    _require_cuda('top_count', top_count, x.dtype)
    want = (s.R, output_dim, pooled_size, pooled_size)
    if tuple(out_grad.shape) != want or tuple(top_count.shape) != want:
        raise RuntimeError(f'out_grad and top_count must be {want}, got {tuple(out_grad.shape)} and '
                           f'{tuple(top_count.shape)}')
    gout, cnt = out_grad.contiguous(), top_count.contiguous()
    sfx = _DTYPE_SFX[x.dtype]
    det = deterministic()
    with torch.cuda.device(x.device):
        grad_trans = torch.zeros_like(trans) if tr is None else torch.zeros_like(tr)
        if not det or tr is not None:
            # grad_trans (and, unless deterministic, grad_input) from the backward kernel; in deterministic mode its
            # scattered grad_input goes to a scratch buffer and is discarded
            grad_input = torch.zeros_like(x)
            # 0 bytes is a valid answer here (no_trans needs no workspace), so the query is not checked
            nbytes = _lib.lib().c2m_psroi_pooling_workspace_bytes(s, x.element_size())
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device) if nbytes else None
            _call(f'c2m_psroi_pooling_backward_{sfx}', gout, x, bbox, tr, cnt, s, grad_input,
                  None if tr is None else grad_trans, ws, nbytes)
        if det:
            grad_input = torch.empty_like(x)
            ws = _det_workspace('c2m_psroi_grad_input_det_workspace_bytes', s, s.B * (1 if no_trans else s.num_classes),
                                x.device) if s.R and grad_input.numel() else None
            _call(f'c2m_psroi_pooling_grad_input_det_{sfx}', gout, bbox, tr, cnt, s, grad_input, ws,
                  0 if ws is None else ws.numel())
    return grad_input, grad_trans


# ------------------------------------------------------------------------------------------------
# Grouped deformable convolution, v1 and modulated (`deform_conv_cuda`, mmsr/models/archs/dcn/src)
def _deform_check(input, weight, offset, mask, kernel_h, kernel_w, groups, deformable_group, **more):
    """Validates dtype, channel / kernel shapes, then devices; returns the dtype suffix."""
    if not isinstance(input, torch.Tensor):
        raise TypeError('input must be a Tensor')
    dtype = input.dtype
    if dtype not in _DTYPE_SFX:
        raise RuntimeError(f'deformable convolution supports torch.float32 and torch.float64, got {dtype}')
    if input.dim() != 4:
        raise RuntimeError(f'input must be [B, C, H, W], got shape {tuple(input.shape)}')
    if weight.dim() != 4 or weight.shape[2] != kernel_h or weight.shape[3] != kernel_w:
        raise RuntimeError(f'Input shape and kernel shape wont match: ({kernel_h} x {kernel_w} vs '
                           f'{tuple(weight.shape[2:])}).')
    C, cout = input.shape[1], weight.shape[0]
    if groups < 1 or C != weight.shape[1] * groups:
        raise RuntimeError(f'Input shape and kernel channels wont match: ({C} vs {weight.shape[1]} x {groups} groups).')
    if cout % groups:
        raise RuntimeError(f'output channels ({cout}) must be divisible by groups ({groups})')
    if deformable_group < 1 or C % deformable_group:
        raise RuntimeError(f'input channels ({C}) must be divisible by deformable groups ({deformable_group})')
    tensors = dict(input=input, weight=weight, offset=offset, mask=mask, **more)
    for n, t in tensors.items():
        if t is not None:
            _require_cuda(n, t, dtype)
            if t.device != input.device:
                raise RuntimeError(f'{n} is on {t.device}, input on {input.device}')
    return _DTYPE_SFX[dtype]


def deform_conv_forward(input, weight, offset, mask, bias, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                        dilation_h, dilation_w, groups, deformable_group):
    """Grouped deformable convolution, fp32 or fp64: mask None is DCNv1 (modulation 1), bias None adds nothing.
    weight [Cout, C/groups, kh, kw]; offset [B, 2*dg*kh*kw, Ho, Wo]; mask [B, dg*kh*kw, Ho, Wo].

    A modulated fp32 call with groups == 1 is exactly `_ext.dcn_v2_forward` (dcn_v2_forward above, zero bias when
    bias is None), so eligible 3x3 shapes run on the tensor cores there."""
    sfx = _deform_check(input, weight, offset, mask, kernel_h, kernel_w, groups, deformable_group, bias=bias)
    geom = (kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w)
    Ho, Wo = _deform_out(input, weight, offset, mask, geom, deformable_group, nonempty=True)
    cout = weight.shape[0]
    if bias is not None and tuple(bias.shape) != (cout,):
        raise RuntimeError(f'bias must be [{cout}], got shape {tuple(bias.shape)}')
    if mask is not None and sfx == 'f32' and groups == 1:
        if bias is None:
            bias = torch.zeros(cout, dtype=input.dtype, device=input.device)
        return dcn_v2_forward(input, weight, bias, offset, mask, *geom, deformable_group)
    return _deform_forward(_dense_nchw_or_nhwc(input), weight, offset, mask, bias, Ho, Wo, geom, groups,
                           deformable_group)


def _deform_forward(x, weight, offset, mask, bias, Ho, Wo, geom, groups, deformable_group):
    """The CUDA-core forward (c2m_deform_conv_forward_*) on checked tensors of one dtype; x dense NCHW or channels-last,
    geom = (kh, kw, sh, sw, ph, pw, dh, dw), mask / bias may be None."""
    cout = weight.shape[0]
    out = torch.empty(x.shape[0], cout, Ho, Wo, dtype=x.dtype, device=x.device)
    s = _shape(x, cout, *geom, deformable_group, out)
    offset, weight = offset.contiguous(), weight.contiguous()
    mask = mask.contiguous() if mask is not None else None
    bias = bias.contiguous() if bias is not None else None
    _call(f'c2m_deform_conv_forward_{_DTYPE_SFX[x.dtype]}', x, offset, mask, weight, bias, groups, out, s,
          device=x.device)
    return out


def deform_conv_backward(input, weight, offset, mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                         pad_w, dilation_h, dilation_w, groups, deformable_group, need_input=True, need_weight=True):
    """Gradients of deform_conv_forward -> (grad_input, grad_offset, grad_mask, grad_weight, grad_bias).

    The deformable pieces are libc2m_sm100 kernels and the two GEMMs are grouped torch.matmul over [groups, ...] views
    in full fp32 / fp64 (TF32 off):
        gcol_g = W_g^T gout_g,   grad_W_g = sum_b gout_g col_g^T.
    grad_mask is None when mask is None.  need_input=False skips grad_input / grad_offset / grad_mask (None),
    need_weight=False skips grad_weight / grad_bias (None)."""
    _deform_check(input, weight, offset, mask, kernel_h, kernel_w, groups, deformable_group, grad_output=grad_output)
    x, w = input.contiguous(), weight.contiguous()
    offset, gout = offset.contiguous(), grad_output.contiguous()
    mask = mask.contiguous() if mask is not None else None
    geom = (kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w)
    _deform_out(x, w, offset, mask, geom, deformable_group, grad_output=gout)
    s = _shape(x, w.shape[0], *geom, deformable_group, gout)
    return _deform_backward(x, w, offset, mask, gout, s, groups, need_input, need_weight)


def _deform_backward(x, w, offset, mask, gout, s, groups, need_input, need_weight):
    """deform_conv_backward on checked, contiguous tensors of one dtype and their DcnShape `s`."""
    B, C = x.shape[:2]
    cout = w.shape[0]
    T, P = s.kh * s.kw, gout.shape[2] * gout.shape[3]
    sfx = _DTYPE_SFX[x.dtype]
    G, cin_g, cout_g = groups, C // groups, cout // groups
    grad_input = grad_offset = grad_mask = grad_weight = grad_bias = None
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.cuda.device(x.device):
            wg = w.view(G, cout_g, cin_g * T)
            gg = gout.view(B, G, cout_g, P)
            columns = None
            if need_input:
                gcol = torch.matmul(wg.transpose(1, 2), gg).contiguous()            # [B, G, Cin_g*T, P] = [B, C*T, P]
                grad_offset = torch.empty_like(offset)
                grad_mask = torch.empty_like(mask) if mask is not None else None
                _call(f'c2m_deform_conv_col2im_coord_{sfx}', gcol, x, offset, mask, s, grad_offset, grad_mask)
                grad_input = _col2im(sfx, gcol, offset, mask, s, x)
                columns = gcol                                                      # reuse the buffer
            if need_weight:
                if columns is None:
                    columns = torch.empty(B, C * T, P, dtype=x.dtype, device=x.device)
                _call(f'c2m_deform_conv_im2col_{sfx}', x, offset, mask, s, columns)
                cg = columns.view(B, G, cin_g * T, P)
                grad_weight = torch.matmul(gg, cg.transpose(2, 3)).sum(0).view_as(w)
                grad_bias = gout.sum(dim=(0, 2, 3))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return grad_input, grad_offset, grad_mask, grad_weight, grad_bias
