"""The general-geometry CUDA-core DCN kernels behind `_ext` (-m gpu), against the fp64-accumulating C oracle.

`dcn_fwd_kernel<NO>` (csrc/dcn_v2.cu) serves `_ext.dcn_v2_forward` for every shape the tensor-core kernel does not take
(anything but 3x3/s1/p1/d1 with C/dg % 8 == 0, and everything under C2M_EXT_DCN_TC=0) and `c2m.dcn_v2_fused_forward`
(the module tail when the tensor-core route is refused).  A CTA owns 64 output pixels and 16 NO output channels, with
NO = 1, 2, 4, 8, 16 for Cout <= 16, 32, 64, 128 and above (then ceil(Cout / 256) z-blocks).  It walks K one deformable group at
a time, taps 9 per pass (MAXT) and the group's channels 32 per pass (MAXCB); a sampling table per (tap, pixel) is shared
by the group's channels.  The gather has a second branch for channels-last input (`xs_c == 1`).  The fused entry adds
the pre-offsets (a `pre_offset` tensor, or the index map decoded with any scale and Ref width), the sigmoid of the mask
and an optional LeakyReLU of any slope.

`_ext.dcn_v2_backward` (csrc/dcn_bwd.cu) runs three grid-stride kernels capped at 132 * 16 blocks of 256 threads
(540 672 threads): `dcn_im2col_kernel` (one thread per (b, c, p)), `dcn_col2im_coord_kernel` (per (b, group, tap, p))
and `dcn_col2im_kernel` (per (b, c, tap, p)), between two fp32 GEMMs that must not run in TF32.  `offset_pyramid_kernel`
(csrc/offsets.cu) caps its grid at 1024 blocks per (tap, image) plane, so maps above 262 144 pixels take the stride.

Case ids name what each case pins:
- `k{kh}x{kw}_s{sh}x{sw}_p{ph}x{pw}_d{dh}x{dw}`: the geometry; every pair is unequal in some case, and `p` larger than
  the kernel's reach with `zero` offsets leaves some outputs with every tap outside the image.
- `Co{Cout}_NO{NO}[x{z-blocks}][-part]`: the instantiation and whether its last channel group / z-block is partial.
- `taps{passes}`: the tap passes (`9+6`, `5x9+4`); `cb{passes}`: the channel passes of one group (`32+1`).
- `nchw`, `cl` (channels-last input, the `xs_c == 1` gather) or `strided` (a non-dense `x[:, :, ::2]` view).
- `bnd`: sampling points placed exactly on -1, -1 + 2^-7, 0, H-1, H-1 + 2^-7, H - 2^-7, H and beyond (the same for w),
  mixed with exact integers and random fractions.  They are dyadic, so `base + offset` is exact in fp32 and kernel and
  oracle take the same branch; unlike tests against autograd, no jitter away from integers is needed.
Masks hold exact zeros, negative values and values above 1: the `_ext` contract takes any modulation.

Bars: 1e-5 of the output scale (forward) and 1e-5 of each gradient's own largest magnitude (backward).  The offset
pyramid and the two pre-offset sources of the fused kernel must match bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle, ref_path

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
MAXT, MAXCB = 9, 32                          # taps and channels per pass of dcn_fwd_kernel


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


def _within(got, want, bar, what=''):
    """max |got - want| <= bar * max |want|; returns the error as a fraction of the bar."""
    want = want.double()
    err = float((got.detach().cpu().double() - want).abs().max())
    scale = float(want.abs().max())
    assert scale > 0, what
    assert err <= bar * scale, f'{what}: max abs err {err:.3e} vs scale {scale:.3e}'
    return err / (bar * scale)


def _refuse_tensor_cores(monkeypatch):
    """Fail the test if anything reaches the tensor-core DCN kernel."""
    from c2m_b200 import ops

    def refuse(*args, **kwargs):
        raise AssertionError('the tensor-core DCN kernel was called')
    monkeypatch.setattr(ops, 'dcn_v2_fused_tc', refuse)


def _ffma_only(monkeypatch):
    """Route every `_ext.dcn_v2_forward` to the FFMA kernel and fail if the tensor-core kernel is reached."""
    monkeypatch.setenv('C2M_EXT_DCN_TC', '0')
    _refuse_tensor_cores(monkeypatch)


def _out_hw(geo, H, W):
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


_EPS = 2.0 ** -7


def _offsets(seed, B, dg, geo, H, W, kind):
    """Offsets [B, 2 dg kh kw, Ho, Wo].  `zero`: all zero.  `bnd`: each of h_im and w_im is independently a boundary
    target (-1, -1 + 2^-7, 0, n-1, n-1 + 2^-7, n - 2^-7, n, n + 1.5), an exact integer in [-2, n+1] or the base position
    plus a random fraction."""
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    Ho, Wo = _out_hw(geo, H, W)
    T = kh * kw
    shape = (B, dg, T, Ho, Wo)
    if kind == 'zero':
        return torch.zeros(B, 2 * dg * T, Ho, Wo)
    rng = np.random.default_rng(seed)
    taps = np.arange(T)
    base_h = (np.arange(Ho) * sh - ph)[None, None, None, :, None] + ((taps // kw) * dh)[None, None, :, None, None]
    base_w = (np.arange(Wo) * sw - pw)[None, None, None, None, :] + ((taps % kw) * dw)[None, None, :, None, None]

    def axis(base, n):
        base = np.broadcast_to(base, shape).astype(np.float64)
        targets = np.array([-1.0, -1.0 + _EPS, 0.0, n - 1.0, n - 1.0 + _EPS, n - _EPS, float(n), n + 1.5])
        pick = rng.integers(0, 3, shape)
        tgt = np.where(pick == 0, targets[rng.integers(0, len(targets), shape)],
                       rng.integers(-2, n + 2, shape).astype(np.float64))
        off = np.where(pick == 2, rng.standard_normal(shape) * 2.0, tgt - base).astype(np.float32)
        exact = pick != 2
        assert np.array_equal((base.astype(np.float32) + off)[exact], tgt[exact].astype(np.float32))
        return off
    off = np.stack([axis(base_h, H), axis(base_w, W)], axis=3)           # [B, dg, T, 2, Ho, Wo]: (h, w) per tap
    return torch.from_numpy(np.ascontiguousarray(off.reshape(B, 2 * dg * T, Ho, Wo)))


def _mask(seed, shape):
    """Modulation with exact zeros, negative values and values above 1."""
    rng = np.random.default_rng(seed)
    m = rng.standard_normal(shape) * 0.8 + 0.4
    m[rng.random(shape) < 0.15] = 0.0
    return torch.from_numpy(m.astype(np.float32))


def _no(cout):
    return 1 if cout <= 16 else 2 if cout <= 32 else 4 if cout <= 64 else 8 if cout <= 128 else 16


def _passes(n, per):
    full, rem = divmod(n, per)
    if full == 0:
        return f'{rem}'
    head = f'{per}' if full == 1 else f'{full}x{per}'
    return head + (f'+{rem}' if rem else '')


def _geo_id(geo):
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    return f'k{kh}x{kw}_s{sh}x{sw}_p{ph}x{pw}_d{dh}x{dw}'


# ------------------------------------------------------------------------------------------- a) FFMA forward
# (geometry (kh, kw, sh, sw, ph, pw, dh, dw), B, C, dg, Cout, H, W, input layout, offsets)
FFMA_CASES = [
    ((1, 1, 2, 1, 2, 1, 1, 1), 2, 3, 3, 5, 9, 7, 'nchw', 'zero'),
    ((1, 1, 1, 1, 0, 0, 1, 1), 1, 33, 1, 300, 10, 13, 'cl', 'bnd'),
    ((2, 2, 1, 1, 0, 0, 1, 1), 3, 6, 2, 16, 11, 13, 'cl', 'bnd'),
    ((1, 3, 1, 1, 0, 1, 1, 1), 2, 32, 1, 24, 10, 12, 'nchw', 'bnd'),
    ((3, 5, 2, 1, 1, 2, 1, 2), 1, 12, 3, 32, 13, 11, 'nchw', 'bnd'),
    ((5, 3, 1, 2, 2, 0, 3, 1), 2, 33, 1, 33, 15, 10, 'cl', 'bnd'),
    ((3, 1, 1, 3, 0, 2, 2, 1), 1, 130, 2, 64, 12, 14, 'nchw', 'bnd'),
    ((5, 5, 2, 2, 1, 1, 1, 1), 2, 40, 1, 65, 12, 11, 'strided', 'bnd'),
    ((7, 7, 1, 1, 3, 3, 1, 1), 1, 80, 2, 128, 9, 10, 'cl', 'bnd'),
    ((3, 3, 1, 1, 1, 1, 1, 1), 2, 64, 2, 129, 13, 17, 'nchw', 'bnd'),     # tensor-core eligible: C2M_EXT_DCN_TC=0
    ((3, 3, 1, 1, 3, 3, 1, 1), 1, 3, 1, 256, 8, 6, 'nchw', 'zero'),
    ((5, 5, 1, 1, 0, 0, 1, 1), 3, 4, 4, 257, 5, 5, 'nchw', 'bnd'),       # 1x1 output map
]


def _ffma_id(c):
    geo, B, C, dg, Cout, H, W, layout, offs = c
    Ho, Wo = _out_hw(geo, H, W)
    no = _no(Cout)
    nz = -(-Cout // (16 * no))
    cpg = C // dg
    return (f'{_geo_id(geo)}_B{B}_C{C}dg{dg}_Co{Cout}_NO{no}{f"x{nz}" if nz > 1 else ""}'
            f'{"-part" if Cout % (16 * no) else ""}_taps{_passes(geo[0] * geo[1], MAXT)}_cb{_passes(cpg, MAXCB)}'
            f'_out{Ho}x{Wo}_{layout}_{offs}')


def _ffma_inputs(case, seed):
    geo, B, C, dg, Cout, H, W, layout, offs = case
    kh, kw = geo[:2]
    Ho, Wo = _out_hw(geo, H, W)
    x = seeding.randn(seed, (B, C, 2 * H if layout == 'strided' else H, W))
    wgt = seeding.randn(seed + 1, (Cout, C, kh, kw), 1.0 / np.sqrt(C * kh * kw))
    bias = seeding.randn(seed + 2, (Cout,))
    off = _offsets(seed + 3, B, dg, geo, H, W, offs)
    mask = _mask(seed + 4, (B, dg * kh * kw, Ho, Wo))
    return x, wgt, bias, off, mask


def _device_input(x, layout):
    xd = x.to(DEV)
    if layout == 'cl':
        xd = xd.contiguous(memory_format=torch.channels_last)
        assert xd.stride(1) == 1
    elif layout == 'strided':
        xd = xd[:, :, ::2]
        assert not xd.is_contiguous()
    return xd


def _host_input(x, layout):
    return x[:, :, ::2].contiguous() if layout == 'strided' else x


@pytest.mark.parametrize('case', FFMA_CASES, ids=_ffma_id)
def test_ext_dcn_forward_ffma_general_geometry_vs_fp64(case, monkeypatch):
    import _ext
    from c2m_b200 import ops
    _ffma_only(monkeypatch)
    geo, B, C, dg, Cout, H, W, layout, offs = case
    x, wgt, bias, off, mask = _ffma_inputs(case, 1000 + FFMA_CASES.index(case) * 10)
    want = c_oracle.dcn_v2_forward(_host_input(x, layout), wgt, bias, off, mask, *geo, dg=dg, acc64=True)
    n0 = ops.launch_count()
    got = _ext.dcn_v2_forward(_device_input(x, layout), wgt.to(DEV), bias.to(DEV), off.to(DEV), mask.to(DEV), *geo, dg)
    assert ops.launch_count() - n0 == 1
    assert got.shape == want.shape and got.is_contiguous()
    _within(got, want, 1e-5, 'forward')


@pytest.mark.parametrize('case', [c for c in FFMA_CASES if c[1] == 3], ids=_ffma_id)
def test_ext_dcn_forward_ffma_batch_equals_single_images_bitwise(case, monkeypatch):
    """Images of a batch are grid rows of the same kernel: running one alone must not change a bit."""
    import _ext
    _ffma_only(monkeypatch)
    geo, B, C, dg, Cout, H, W, layout, offs = case
    x, wgt, bias, off, mask = _ffma_inputs(case, 2000)
    xd = _device_input(x, layout)
    wgt, bias, off, mask = [t.to(DEV) for t in (wgt, bias, off, mask)]
    full = _ext.dcn_v2_forward(xd, wgt, bias, off, mask, *geo, dg)
    for i in range(B):
        one = _ext.dcn_v2_forward(xd[i:i + 1], wgt, bias, off[i:i + 1], mask[i:i + 1], *geo, dg)
        assert torch.equal(full[i:i + 1], one), i


def test_ext_dcn_shape_checks_use_each_axis():
    """Offsets shaped for the transposed kernel, or for the other axis' stride, are refused before any launch."""
    import _ext
    z = lambda *s: torch.zeros(*s, device=DEV)
    x, w, b = z(1, 4, 11, 10), z(6, 4, 3, 5), z(6)
    Ho, Wo = _out_hw((3, 5, 2, 1, 1, 2, 1, 2), 11, 10)
    assert (Ho, Wo) == (6, 6)
    Ho2, Wo2 = _out_hw((3, 5, 1, 2, 1, 2, 1, 2), 11, 10)
    with pytest.raises(RuntimeError, match='mismatch'):
        _ext.dcn_v2_forward(x, w, b, z(1, 30, Ho2, Wo2), z(1, 15, Ho2, Wo2), 3, 5, 2, 1, 1, 2, 1, 2, 1)
    with pytest.raises(RuntimeError, match='kernel shape wont match'):
        _ext.dcn_v2_forward(x, w, b, z(1, 30, Ho, Wo), z(1, 15, Ho, Wo), 5, 3, 2, 1, 1, 2, 1, 2, 1)
    with pytest.raises(RuntimeError, match='grad_output has shape'):
        _ext.dcn_v2_backward(x, w, b, z(1, 30, Ho, Wo), z(1, 15, Ho, Wo), z(1, 6, Ho2, Wo2), 3, 5, 2, 1, 1, 2, 1, 2, 1)


# ------------------------------------------------------------------------------------------- b) fused CUDA-core forward
# (B, C, dg, Cout, scale, gh, gw, ref_gw, pre-offset source, lrelu slope, bias, channels-last output); H = s (gh + 2)
FUSED_CASES = [
    (2, 3, 1, 16, 1, 9, 13, None, 'idx', 1.0, True, False),
    (1, 10, 2, 24, 2, 6, 5, 9, 'idx', 0.2, False, True),
    (2, 36, 3, 40, 3, 5, 4, None, 'idx', 0.1, True, False),
    (1, 80, 2, 33, 4, 3, 4, 6, 'pre', 0.2, True, True),
    (1, 40, 8, 20, 2, 7, 5, 11, 'pre', 1.0, False, False),
]


def _fused_id(c):
    B, C, dg, Cout, s, gh, gw, ref_gw, src, slope, has_bias, cl = c
    return (f'C{C}dg{dg}_Co{Cout}_NO{_no(Cout)}_{src}-s{s}{f"-refgw{ref_gw}" if ref_gw else ""}_slope{slope:g}'
            f'{"" if has_bias else "_nobias"}{"_clout" if cl else ""}_B{B}_{s * (gh + 2)}x{s * (gw + 2)}')


def _index_map(seed, B, gh, gw, ref_gw):
    """Random index map into a Ref grid of (gh + 1) rows of ref_gw (default gw) patches."""
    return torch.from_numpy(np.random.default_rng(seed).integers(0, (gh + 1) * (ref_gw or gw), (B, gh, gw)))


def _fused_inputs(case, seed):
    B, C, dg, Cout, s, gh, gw, ref_gw, src, slope, has_bias, cl = case
    H, W = s * (gh + 2), s * (gw + 2)
    x = seeding.randn(seed, (B, C, H, W))
    om = seeding.randn(seed + 1, (B, 27 * dg, H, W), 0.7)
    wgt = seeding.randn(seed + 2, (Cout, C, 3, 3), 1.0 / np.sqrt(9 * C))
    bias = seeding.randn(seed + 3, (Cout,)) if has_bias else None
    idx = _index_map(seed + 4, B, gh, gw, ref_gw)
    return x, om, wgt, bias, idx


def _pyramid_oracle(idx, s, ref_gw):
    return torch.stack([c_oracle.offset_pyramid(idx[b], s, ref_gw) for b in range(idx.shape[0])])


def _fused_oracle(x, om, wgt, bias, dg, pre, slope):
    """The module tail in the reference's formulation: om offsets + the (x, y) pyramid reordered to (h, w) pairs,
    sigmoid mask, the literal DCN, then LeakyReLU."""
    n = dg * 9
    off = om[:, :2 * n].clone()
    pr = pre.repeat(1, dg, 1, 1, 1)
    off[:, 0::2] += pr[..., 1]
    off[:, 1::2] += pr[..., 0]
    bias = bias if bias is not None else torch.zeros(wgt.shape[0])
    want = c_oracle.dcn_v2_forward(x, wgt, bias, off, torch.sigmoid(om[:, 2 * n:]), dg=dg, acc64=True)
    return want if slope == 1.0 else F.leaky_relu(want, slope)


@pytest.mark.parametrize('case', FUSED_CASES, ids=_fused_id)
def test_dcn_fused_forward_vs_fp64(case):
    import c2m_b200 as c2m
    B, C, dg, Cout, s, gh, gw, ref_gw, src, slope, has_bias, cl = case
    x, om, wgt, bias, idx = _fused_inputs(case, 3000 + FUSED_CASES.index(case) * 10)
    pre = _pyramid_oracle(idx, s, ref_gw)
    want = _fused_oracle(x, om, wgt, bias, dg, pre, slope)
    kw = dict(idx=idx.to(DEV), pre_scale=s, ref_gw=ref_gw) if src == 'idx' else dict(pre_offset=pre.to(DEV))
    got = c2m.dcn_v2_fused_forward(x.to(DEV), om.to(DEV), wgt.to(DEV), bias.to(DEV) if has_bias else None, dg,
                                   lrelu_slope=slope, channels_last_out=cl, **kw)
    assert got.is_contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
    _within(got, want, 1e-5, 'fused forward')


@pytest.mark.parametrize('case', FUSED_CASES, ids=_fused_id)
def test_dcn_fused_forward_idx_decode_equals_pre_offset_bitwise(case):
    """The in-kernel index-map decode and the materialised pyramid add the same integer-valued floats in the same order."""
    import c2m_b200 as c2m
    B, C, dg, Cout, s, gh, gw, ref_gw, src, slope, has_bias, cl = case
    x, om, wgt, bias, idx = [t.to(DEV) if t is not None else None for t in _fused_inputs(case, 4000)]
    pre = c2m.offset_pyramid(idx, s, ref_gw)
    a = c2m.dcn_v2_fused_forward(x, om, wgt, bias, dg, idx=idx, pre_scale=s, ref_gw=ref_gw, lrelu_slope=slope)
    b = c2m.dcn_v2_fused_forward(x, om, wgt, bias, dg, pre_offset=pre, lrelu_slope=slope)
    assert torch.equal(a, b)


def test_dcn_sep_pre_multi_offset_lrelu02_takes_cuda_core_route(monkeypatch):
    """LeakyReLU slope 0.2 is not fused by the tensor-core kernel, so the model's 64-channel dg = 8 layer runs the
    CUDA-core fused kernel: it must match the oracle on the offsets its own conv_offset_mask produced."""
    from mmsr.models.archs.DCNv2.dcn_v2 import DCN_sep_pre_multi_offset
    _refuse_tensor_cores(monkeypatch)
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    B, C, dg, s, gh, gw = 1, 64, 8, 2, 7, 9
    H, W = s * (gh + 2), s * (gw + 2)
    m = DCN_sep_pre_multi_offset(C, C, 3, stride=1, padding=1, deformable_groups=dg)
    sd = seeding.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, 5100)
    sd['conv_offset_mask.weight'] = sd['conv_offset_mask.weight'] * 3.0
    m.load_state_dict(sd)
    m.to(DEV).eval()
    x = seeding.randn(5101, (B, C, H, W)).to(DEV)
    feat = seeding.randn(5102, (B, C, H, W)).to(DEV)
    idx = _index_map(5103, B, gh, gw, None)
    pre = _pyramid_oracle(idx, s, None)
    with torch.no_grad():
        got = m([x, feat], pre.to(DEV), lrelu_slope=0.2)
        om = m.conv_offset_mask(feat)
    want = _fused_oracle(x.cpu(), om.cpu(), m.weight.detach().cpu(), m.bias.detach().cpu(), dg, pre, 0.2)
    _within(got, want, 1e-5, 'module')


# ------------------------------------------------------------------------------------------- c) backward
# (geometry, B, C, dg, Cout, H, W)
BWD_CASES = [
    ((1, 3, 1, 1, 0, 1, 1, 1), 2, 4, 1, 5, 7, 9),
    ((3, 5, 2, 1, 1, 2, 1, 2), 1, 6, 2, 7, 11, 10),
    ((5, 3, 1, 2, 2, 0, 3, 1), 1, 9, 3, 4, 14, 9),
    ((3, 1, 1, 3, 0, 2, 2, 1), 2, 8, 4, 6, 10, 11),
    ((2, 2, 1, 1, 0, 0, 1, 1), 1, 12, 4, 5, 8, 7),
    ((7, 7, 1, 1, 3, 3, 1, 1), 1, 40, 1, 16, 10, 10),
    ((3, 5, 1, 2, 1, 2, 2, 1), 1, 64, 1, 96, 10, 14),
    ((3, 3, 1, 1, 1, 1, 1, 1), 2, 16, 8, 8, 136, 136),
]
_BWD_CAP = 132 * 16 * 256                    # threads of one pass of the backward kernels' capped grids


def _bwd_id(c):
    geo, B, C, dg, Cout, H, W = c
    Ho, Wo = _out_hw(geo, H, W)
    T, P = geo[0] * geo[1], Ho * Wo
    n = (B * C * P, B * dg * T * P, B * C * T * P)          # threads wanted by im2col, col2im_coord, col2im
    stride = '_gridstride-all3' if min(n) > _BWD_CAP else ''
    return f'{_geo_id(geo)}_B{B}_C{C}dg{dg}_Co{Cout}_{H}x{W}_bnd{stride}'


def _bwd_inputs(case, seed):
    geo, B, C, dg, Cout, H, W = case
    kh, kw = geo[:2]
    Ho, Wo = _out_hw(geo, H, W)
    x = seeding.randn(seed, (B, C, H, W))
    wgt = seeding.randn(seed + 1, (Cout, C, kh, kw), 1.0 / np.sqrt(C * kh * kw))
    bias = seeding.randn(seed + 2, (Cout,))
    off = _offsets(seed + 3, B, dg, geo, H, W, 'bnd')
    mask = _mask(seed + 4, (B, dg * kh * kw, Ho, Wo))
    gout = seeding.randn(seed + 5, (B, Cout, Ho, Wo))
    return x, wgt, bias, off, mask, gout


_GRADS = ('input', 'offset', 'mask', 'weight', 'bias')


@pytest.mark.parametrize('case', BWD_CASES, ids=_bwd_id)
def test_ext_dcn_backward_general_geometry_vs_fp64(case):
    import _ext
    geo, B, C, dg, Cout, H, W = case
    t = _bwd_inputs(case, 6000 + BWD_CASES.index(case) * 10)
    want = c_oracle.dcn_v2_backward(*t, *geo, dg)
    got = _ext.dcn_v2_backward(*[v.to(DEV) for v in t], *geo, dg)
    for g_, w_, name in zip(got, want, _GRADS):
        assert g_.shape == w_.shape, name
        _within(g_, w_, 1e-5, name)


def test_ext_dcn_backward_gemms_ignore_tf32_flag():
    """`dcn_v2_backward` runs its two GEMMs in full fp32 even when the caller allows TF32, and gives the flag back."""
    import _ext
    case = BWD_CASES[6]
    geo, B, C, dg, Cout, H, W = case
    t = _bwd_inputs(case, 7000)
    want = c_oracle.dcn_v2_backward(*t, *geo, dg)
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = True
        got = _ext.dcn_v2_backward(*[v.to(DEV) for v in t], *geo, dg)
        assert torch.backends.cuda.matmul.allow_tf32 is True
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    for g_, w_, name in zip(got, want, _GRADS):
        _within(g_, w_, 1e-5, name)


# ------------------------------------------------------------------------------------------- d) modules, tuple geometry
def test_dcnv2_autograd_tuple_geometry_vs_fp64(monkeypatch):
    """`_DCNv2` hands (kh, kw), (sh, sw), (ph, pw), (dh, dw) to forward and backward in the right order."""
    from mmsr.models.archs.DCNv2.dcn_v2 import DCNv2
    _ffma_only(monkeypatch)
    geo = (3, 5, 2, 1, 1, 2, 1, 2)
    B, C, Cout, dg, H, W = 2, 6, 10, 2, 11, 10
    Ho, Wo = _out_hw(geo, H, W)
    m = DCNv2(C, Cout, kernel_size=(3, 5), stride=(2, 1), padding=(1, 2), dilation=(1, 2), deformable_groups=dg)
    with torch.no_grad():
        m.weight.copy_(seeding.randn(8001, (Cout, C, 3, 5), 0.2))
        m.bias.copy_(seeding.randn(8002, (Cout,)))
    m.to(DEV)
    x = seeding.randn(8003, (B, C, H, W))
    off = _offsets(8004, B, dg, geo, H, W, 'bnd')
    mask = _mask(8005, (B, dg * 15, Ho, Wo))
    g = seeding.randn(8006, (B, Cout, Ho, Wo))
    leaves = [t.to(DEV).requires_grad_(True) for t in (x, off, mask)]
    y = m(*leaves)
    w_cpu, b_cpu = m.weight.detach().cpu(), m.bias.detach().cpu()
    _within(y, c_oracle.dcn_v2_forward(x, w_cpu, b_cpu, off, mask, *geo, dg=dg, acc64=True), 1e-5, 'forward')
    y.backward(g.to(DEV))
    want = c_oracle.dcn_v2_backward(x, w_cpu, b_cpu, off, mask, g, *geo, dg)
    for got, w_, name in zip((leaves[0].grad, leaves[1].grad, leaves[2].grad, m.weight.grad, m.bias.grad), want, _GRADS):
        _within(got, w_, 1e-5, name)


@pytest.mark.parametrize('variant', ['DCN_k3x5_s2x1_p1x2_dg2', 'DCN_sep_k5x3_s1x1_p2x1_dg4'])
def test_dcn_modules_non_square_kernel_equal_ext(variant, monkeypatch):
    """DCN / DCN_sep with a non-square kernel == `_ext.dcn_v2_forward` on the offsets and mask their own
    conv_offset_mask produced."""
    import _ext
    from mmsr.models.archs.DCNv2.dcn_v2 import DCN, DCN_sep
    _ffma_only(monkeypatch)
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    C, Cout, H, W = 8, 12, 13, 11
    if variant.startswith('DCN_sep'):
        m, geo, dg = DCN_sep(C, Cout, kernel_size=(5, 3), stride=1, padding=(2, 1), deformable_groups=4), (5, 3, 1, 1, 2, 1, 1, 1), 4
    else:
        m, geo, dg = DCN(C, Cout, kernel_size=(3, 5), stride=(2, 1), padding=(1, 2), deformable_groups=2), (3, 5, 2, 1, 1, 2, 1, 1), 2
    sd = seeding.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, 8100)
    sd['conv_offset_mask.weight'] = sd['conv_offset_mask.weight'] * 4.0
    m.load_state_dict(sd)
    m.to(DEV).eval()
    x = seeding.randn(8101, (2, C, H, W)).to(DEV)
    feat = seeding.randn(8102, (2, C, H, W)).to(DEV)
    with torch.no_grad():
        if variant.startswith('DCN_sep'):
            y = m([x, feat])
            off, mask = m._offset_mask(feat)
        else:
            y = m(x)
            off, mask = m._offset_mask(x)
        assert tuple(y.shape[2:]) == _out_hw(geo, H, W) == tuple(off.shape[2:])
        want = _ext.dcn_v2_forward(x, m.weight, m.bias, off.contiguous(), mask.contiguous(), *geo, dg)
    assert float(off.abs().max()) > 1.0
    assert torch.equal(y, want)


# ------------------------------------------------------------------------------------------- f) offset pyramid
# (gh, gw, scale, ref_gw)
PYRAMID_CASES = [(158, 158, 4, None), (9, 14, 3, 17), (40, 31, 1, 29), (20, 20, 2, None)]
_PYR_CAP = 1024 * 256


def _pyr_id(c):
    gh, gw, s, ref_gw = c
    n = s * (gh + 2) * s * (gw + 2)
    return f'gh{gh}_gw{gw}_s{s}{f"_refgw{ref_gw}" if ref_gw else ""}_px{n}{"_gridstride" if n > _PYR_CAP else ""}'


@pytest.mark.parametrize('case', PYRAMID_CASES, ids=_pyr_id)
def test_offset_pyramid_vs_oracle_bitwise(case):
    import c2m_b200 as c2m
    gh, gw, s, ref_gw = case
    idx = _index_map(9000 + s, 2, gh, gw, ref_gw)
    got = c2m.offset_pyramid(idx.to(DEV), s, ref_gw).cpu()
    assert torch.equal(got, _pyramid_oracle(idx, s, ref_gw))
    if ref_gw is None and s in (1, 2, 4):
        # the reference's own rule (index_to_flow + shifted, upsampled copies), which decodes with the input width
        key = {1: 'relu3_1', 2: 'relu2_1', 4: 'relu1_1'}[s]
        for b in range(2):
            assert torch.equal(got[b], ref_path.offset_pyramid(ref_path.index_to_flow(idx[b]))[key]), b
