"""Grouped deformable convolution behind `mmsr.models.archs.dcn` (-m gpu), against the C oracle
(oracle/deform_conv_oracle.c, pinned against torchvision's fp64 autograd by tests/test_deform_conv_oracle.py).

`dcn_fwd_kernel<T, NO>` (csrc/dcn_v2.cu) gives each CTA 16 NO output channels of one conv group, with NO chosen from
Cout_g = Cout / groups (fp64 stops at NO = 8), and walks the conv group's input channels in segments that never cross a
deformable-group boundary: taps 9 per pass, channels 32 (fp32) or 16 (fp64) per pass.  The backward kernels
(csrc/dcn_bwd.cu) do not see conv groups; the two GEMMs around them are grouped torch.matmul calls.

Case ids name what each case pins: the geometry `k{kh}x{kw}_s.._p.._d..` (every pair unequal in some case), `g{groups}`
and `dg{dg}` (misaligned when dg does not divide into or out of groups), `Cog{Cout_g}` (partial NO blocks), `taps` and
`cb` passes.  Offsets use the dyadic `bnd` construction of test_gpu_dcn_general.py (sampling points exactly on the
image border, exact in both dtypes, so kernel and oracle take the same branch); masks hold exact zeros, negative values
and values above 1.

Bars: fp32 1e-5 of the output scale (forward) and of each gradient's own largest magnitude; fp64 1e-11 (forward) and
1e-10 (gradients).  Shapes on the tensor-core route use the `_ext` tensor-core bar (2e-5 of the output scale)."""
import numpy as np
import pytest
import torch

import seeding
from oracle import deform_conv_oracle as dco
from test_gpu_dcn_general import _mask, _offsets

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32, F64 = torch.float32, torch.float64
FWD_BAR = {F32: 1e-5, F64: 1e-11}
BWD_BAR = {F32: 1e-5, F64: 1e-10}
_worst = {}                                  # largest error as a fraction of its bar, per (check, dtype)


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    yield
    if _worst:
        print('\ndeform_conv: largest error / bar: ' + ', '.join(f'{k} {v:.3f}' for k, v in sorted(_worst.items())))


def _within(got, want, bar, what):
    want = want.double()
    err = float((got.detach().cpu().double() - want).abs().max())
    scale = float(want.abs().max())
    assert scale > 0, what
    assert err <= bar * scale, f'{what}: max abs err {err:.3e} vs scale {scale:.3e}'
    frac = err / (bar * scale)
    key = what.split(':')[0]
    _worst[key] = max(_worst.get(key, 0.0), frac)
    return frac


def _out_hw(geo, H, W):
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def _passes(n, per):
    full, rem = divmod(n, per)
    return f'{rem}' if full == 0 else (f'{per}' if full == 1 else f'{full}x{per}') + (f'+{rem}' if rem else '')


# (geometry (kh, kw, sh, sw, ph, pw, dh, dw), B, C, Cout, groups, dg, H, W)
CASES = [
    ((3, 3, 1, 1, 1, 1, 1, 1), 2, 6, 6, 3, 2, 9, 8),           # C = 6, groups = 3, dg = 2: a group split by dg
    ((3, 5, 2, 1, 1, 2, 1, 2), 1, 8, 10, 2, 4, 11, 10),
    ((5, 5, 1, 1, 2, 2, 1, 1), 2, 12, 20, 4, 3, 9, 9),         # taps 9+9+7
    ((3, 3, 1, 1, 1, 1, 1, 1), 1, 64, 64, 32, 4, 12, 13),      # groups = 32
    ((3, 1, 1, 3, 0, 2, 2, 1), 1, 96, 40, 2, 1, 10, 11),       # 48 channels per conv group: channel passes 32+16 / 3x16
    ((1, 3, 1, 2, 0, 1, 1, 1), 2, 30, 36, 3, 5, 8, 12),        # dg 5 against groups 3
    ((5, 3, 1, 2, 2, 0, 3, 1), 1, 16, 300, 1, 2, 13, 8),       # groups 1, Cout 300: NO = 16 (fp32) / 8 x 3 (fp64)
    ((2, 2, 1, 1, 0, 0, 1, 1), 3, 9, 6, 3, 3, 8, 7),
]


def _case_id(c):
    geo, B, C, Cout, groups, dg, H, W = c
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    cin_g, cpg = C // groups, C // dg
    seg = min(cin_g, cpg)
    return (f'k{kh}x{kw}_s{sh}x{sw}_p{ph}x{pw}_d{dh}x{dw}_B{B}_C{C}_g{groups}_dg{dg}_Cog{Cout // groups}'
            f'_taps{_passes(kh * kw, 9)}_cb{_passes(seg, 32)}_{H}x{W}')


def _inputs(case, seed, modulated, dtype):
    geo, B, C, Cout, groups, dg, H, W = case
    kh, kw = geo[:2]
    Ho, Wo = _out_hw(geo, H, W)
    x = seeding.randn(seed, (B, C, H, W))
    wgt = seeding.randn(seed + 1, (Cout, C // groups, kh, kw), 1.0 / np.sqrt(C // groups * kh * kw))
    bias = seeding.randn(seed + 2, (Cout,)) if modulated else None
    off = _offsets(seed + 3, B, dg, geo, H, W, 'bnd')
    mask = _mask(seed + 4, (B, dg * kh * kw, Ho, Wo)) if modulated else None
    gout = seeding.randn(seed + 5, (B, Cout, Ho, Wo))
    return [t.to(dtype) if t is not None else None for t in (x, wgt, bias, off, mask, gout)]


def _dev(*ts):
    return [t.to(DEV) if t is not None else None for t in ts]


def _symmetric(geo):
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    return sh == sw and ph == pw and dh == dw


def _forward(case, x, wgt, bias, off, mask, modulated):
    """Through the module-level Functions; a modulated case with per-axis geometry goes through the
    deform_conv_cuda boundary (the modulated Function takes one int per stride / padding / dilation)."""
    from mmsr.models.archs.dcn import deform_conv, deform_conv_cuda, modulated_deform_conv
    geo, B, C, Cout, groups, dg, H, W = case
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    if not modulated:
        return deform_conv(x, off, wgt, (sh, sw), (ph, pw), (dh, dw), groups, dg)
    if _symmetric(geo):
        return modulated_deform_conv(x, off, mask, wgt, bias, sh, ph, dh, groups, dg)
    out = x.new_empty(B, Cout, *_out_hw(geo, H, W))
    deform_conv_cuda.modulated_deform_conv_cuda_forward(x, wgt, bias, None, off, mask, out, None, kh, kw, sh, sw, ph,
                                                        pw, dh, dw, groups, dg, True)
    return out


def _tc_route(case, modulated, dtype):
    from c2m_b200 import ops
    geo, B, C, Cout, groups, dg, H, W = case
    return (modulated and dtype == F32 and groups == 1 and geo == (3, 3, 1, 1, 1, 1, 1, 1)
            and ops.dcn_tc_supported(C, Cout, dg))


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('modulated', [False, True], ids=['v1', 'modulated'])
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_deform_conv_forward_vs_oracle(case, modulated, dtype):
    from c2m_b200 import ops
    geo, B, C, Cout, groups, dg, H, W = case
    x, wgt, bias, off, mask, _ = _inputs(case, 100 + 10 * CASES.index(case), modulated, dtype)
    want = dco.forward(x, wgt, bias, off, mask, *geo, groups, dg)
    n0 = ops.launch_count()
    got = _forward(case, *_dev(x, wgt, bias, off, mask), modulated)
    assert ops.launch_count() - n0 == 1
    assert got.dtype == dtype and got.shape == want.shape
    _within(got, want, 2e-5 if _tc_route(case, modulated, dtype) else FWD_BAR[dtype], f'forward:{dtype}')


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('modulated', [False, True], ids=['v1', 'modulated'])
@pytest.mark.parametrize('case', [CASES[i] for i in (0, 1, 2, 4, 5, 7)], ids=_case_id)
def test_deform_conv_backward_vs_oracle(case, modulated, dtype):
    """Every gradient of both Functions through autograd (a modulated case with per-axis geometry through the
    deform_conv_cuda boundary's backward, on zeroed gradient tensors)."""
    from mmsr.models.archs.dcn import deform_conv_cuda
    geo, B, C, Cout, groups, dg, H, W = case
    x, wgt, bias, off, mask, gout = _inputs(case, 200 + 10 * CASES.index(case), modulated, dtype)
    want = dco.backward(x, wgt, off, mask, gout, *geo, groups, dg)
    if modulated and not _symmetric(geo):
        xd, wd, bd, od, md, gd = _dev(x, wgt, bias, off, mask, gout)
        got = [torch.zeros_like(t) for t in (xd, od, md, wd, bd)]
        deform_conv_cuda.modulated_deform_conv_cuda_backward(xd, wd, bd, None, od, md, None, got[0], got[3], got[4],
                                                             got[1], got[2], gd, *geo, groups, dg, True)
    else:
        leaves = [t.to(DEV).requires_grad_(True) if t is not None else None for t in (x, wgt, bias, off, mask)]
        y = _forward(case, *leaves, modulated)
        y.backward(gout.to(DEV))
        got = (leaves[0].grad, leaves[3].grad, leaves[4].grad if modulated else None, leaves[1].grad,
               leaves[2].grad if modulated else None)
    for g_, w_, name in zip(got, want, ('input', 'offset', 'mask', 'weight', 'bias')):
        if name in ('mask', 'bias') and not modulated:
            continue
        assert g_.dtype == dtype, name
        _within(g_, w_, BWD_BAR[dtype], f'backward:{dtype}:{name}')


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
def test_deform_conv_cuda_inplace_contract(dtype):
    """Accumulating outputs add to what the caller passed, overwritten ones are replaced, gradWeight takes `scale`."""
    from mmsr.models.archs.dcn import deform_conv_cuda as dc
    case = CASES[1]
    geo, B, C, Cout, groups, dg, H, W = case
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    x, wgt, bias, off, mask, gout = _dev(*_inputs(case, 300, True, dtype))
    xc, wc, bc, oc, mc, gc = [t.cpu() for t in (x, wgt, bias, off, mask, gout)]
    gi0, gw0, gb0 = [seeding.randn(301 + i, tuple(t.shape)).to(dtype) for i, t in enumerate((x, wgt, bias))]
    junk = lambda t: torch.full_like(t, 7.0)
    bar = BWD_BAR[dtype]

    # v1
    gx1, goff1, _, gw1, _ = dco.backward(xc, wc, oc, None, gc, *geo, groups, dg)
    gi, go = gi0.to(DEV), junk(off)
    assert dc.deform_conv_backward_input_cuda(x, off, gout, gi, go, wgt, None, kw, kh, sw, sh, pw, ph, dw, dh, groups,
                                              dg, B) == 1
    _within(gi, gi0 + gx1, bar, f'inplace:{dtype}:v1 gradInput')
    _within(go, goff1, bar, f'inplace:{dtype}:v1 gradOffset')
    gw = gw0.to(DEV)
    dc.deform_conv_backward_parameters_cuda(x, off, gout, gw, None, None, kw, kh, sw, sh, pw, ph, dw, dh, groups, dg,
                                            0.25, 1)
    _within(gw, gw0 + 0.25 * gw1, bar, f'inplace:{dtype}:v1 gradWeight')
    out = junk(gout)
    dc.deform_conv_forward_cuda(x, wgt, off, out, None, None, kw, kh, sw, sh, pw, ph, dw, dh, groups, dg, 1)
    _within(out, dco.forward(xc, wc, None, oc, None, *geo, groups, dg), FWD_BAR[dtype], f'inplace:{dtype}:v1 output')

    # modulated
    gx2, goff2, gm2, gw2, gb2 = dco.backward(xc, wc, oc, mc, gc, *geo, groups, dg)
    gi, gw, gb, go, gm = gi0.to(DEV), gw0.to(DEV), gb0.to(DEV), junk(off), junk(mask)
    dc.modulated_deform_conv_cuda_backward(x, wgt, bias, None, off, mask, None, gi, gw, gb, go, gm, gout, kh, kw, sh,
                                           sw, ph, pw, dh, dw, groups, dg, True)
    for got, want, name in ((gi, gi0 + gx2, 'grad_input'), (gw, gw0 + gw2, 'grad_weight'), (gb, gb0 + gb2, 'grad_bias'),
                            (go, goff2, 'grad_offset'), (gm, gm2, 'grad_mask')):
        _within(got, want, bar, f'inplace:{dtype}:{name}')
    gb = gb0.to(DEV)
    dc.modulated_deform_conv_cuda_backward(x, wgt, bias, None, off, mask, None, gi0.to(DEV), gw0.to(DEV), gb, junk(off),
                                           junk(mask), gout, kh, kw, sh, sw, ph, pw, dh, dw, groups, dg, False)
    assert torch.equal(gb, gb0.to(DEV))               # with_bias False: grad_bias untouched
    out = junk(gout)
    dc.modulated_deform_conv_cuda_forward(x, wgt, bias, None, off, mask, out, None, kh, kw, sh, sw, ph, pw, dh, dw,
                                          groups, dg, False)
    _within(out, dco.forward(xc, wc, None, oc, mc, *geo, groups, dg), FWD_BAR[dtype], f'inplace:{dtype}:no-bias output')


def _smooth_inputs(seed, B, C, Cout, groups, dg, H, W, modulated):
    x = seeding.randn(seed, (B, C, H, W)).double()
    w = seeding.randn(seed + 1, (Cout, C // groups, 3, 3), 0.3).double()
    off = seeding.randn(seed + 2, (B, 18 * dg, H, W), 1.5).double()
    off = torch.where((off - off.round()).abs() < 0.1, off + 0.23, off)     # away from the bilinear kinks
    mask = torch.sigmoid(seeding.randn(seed + 3, (B, 9 * dg, H, W))).double() if modulated else None
    b = seeding.randn(seed + 4, (Cout,)).double() if modulated else None
    return x, w, off, mask, b


def test_gradcheck_fp64_groups2_dg2():
    from mmsr.models.archs.dcn import deform_conv, modulated_deform_conv
    x, w, off, _, _ = _smooth_inputs(400, 1, 4, 4, 2, 2, 5, 6, False)
    ins = [t.to(DEV).requires_grad_(True) for t in (x, off, w)]
    assert torch.autograd.gradcheck(lambda a, o, k: deform_conv(a, o, k, 1, 1, 1, 2, 2), ins, nondet_tol=1e-10)
    x, w, off, mask, b = _smooth_inputs(410, 1, 4, 4, 2, 2, 5, 6, True)
    ins = [t.to(DEV).requires_grad_(True) for t in (x, off, mask, w, b)]
    assert torch.autograd.gradcheck(lambda a, o, m, k, bb: modulated_deform_conv(a, o, m, k, bb, 1, 1, 1, 2, 2), ins,
                                    nondet_tol=1e-10)


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
def test_pack_modules_forward_backward(dtype, monkeypatch):
    """DeformConvPack (the 9-gradient backward) and ModulatedDeformConvPack with grouped weights and non-zero offset
    predictors, against the oracle on the offsets / masks the modules predicted themselves."""
    from mmsr.models.archs.dcn import DeformConvPack, ModulatedDeformConvPack
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    B, C, Cout, H, W = 2, 8, 6, 10, 9
    for cls, kw_ in ((DeformConvPack, dict(groups=2, deformable_groups=4)),
                     (ModulatedDeformConvPack, dict(groups=2, deformable_groups=4))):
        m = cls(C, Cout, 3, stride=1, padding=1, **kw_)
        sd = seeding.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, 500)
        key = 'conv_offset.weight' if cls is DeformConvPack else 'conv_offset_mask.weight'
        sd[key] = sd[key] * 3.0
        m.load_state_dict(sd)
        m.to(DEV, dtype)
        x = seeding.randn(501, (B, C, H, W)).to(DEV, dtype).requires_grad_(True)
        y = m(x)
        loss = (y * y).sum()
        loss.backward()
        assert x.grad is not None and m.weight.grad is not None
        with torch.no_grad():
            if cls is DeformConvPack:
                off, mask, bias = m.conv_offset(x), None, None
            else:
                om = m.conv_offset_mask(x)
                off, mask, bias = om[:, :72], torch.sigmoid(om[:, 72:]), m.bias
        assert float(off.abs().max()) > 1.0
        args = [t.detach().cpu() if t is not None else None for t in (x, m.weight, bias, off, mask)]
        want = dco.forward(*args, 3, 3, 1, 1, 1, 1, 1, 1, 2, 4)
        _within(y, want, FWD_BAR[dtype], f'module:{dtype}:{cls.__name__}')
        gx, _, _, gw, _ = dco.backward(args[0], args[1], args[3], args[4], (2 * y).detach().cpu(), 3, 3, 1, 1, 1, 1,
                                       1, 1, 2, 4)
        _within(m.weight.grad, gw, BWD_BAR[dtype], f'module:{dtype}:{cls.__name__} weight grad')


def test_forward_f32_groups1_mask_equals_ext_bitwise(monkeypatch):
    """The generalised kernel at fp32, groups = 1, mask given is the `_ext` FFMA kernel bit for bit."""
    import _ext
    from c2m_b200 import _lib, ops
    monkeypatch.setenv('C2M_EXT_DCN_TC', '0')
    for case in (CASES[6], ((3, 3, 1, 1, 1, 1, 1, 1), 2, 64, 64, 1, 8, 20, 18), ((1, 3, 1, 2, 0, 1, 1, 1), 1, 40, 33,
                                                                                  1, 1, 8, 12)):
        geo, B, C, Cout, groups, dg, H, W = case
        x, wgt, bias, off, mask, _ = _dev(*_inputs(case, 600, True, F32))
        want = _ext.dcn_v2_forward(x, wgt, bias, off, mask, *geo, dg)
        out = torch.empty_like(want)
        s = ops._shape(x, Cout, *geo, dg, out)
        _lib.check(_lib.lib().c2m_deform_conv_forward_f32(x.data_ptr(), off.data_ptr(), mask.data_ptr(),
                                                          wgt.data_ptr(), bias.data_ptr(), 1, out.data_ptr(), s,
                                                          ops._stream()), 'c2m_deform_conv_forward_f32')
        assert torch.equal(out, want), case
        assert torch.equal(ops.deform_conv_forward(x, wgt, off, mask, bias, *geo, 1, dg), want), case


def test_modulated_eligible_shape_takes_tensor_core_route(monkeypatch):
    from c2m_b200 import ops
    from mmsr.models.archs.dcn import modulated_deform_conv
    calls = []
    real = ops.dcn_v2_fused_tc

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(ops, 'dcn_v2_fused_tc', spy)
    case = ((3, 3, 1, 1, 1, 1, 1, 1), 1, 64, 64, 1, 8, 24, 20)
    geo, B, C, Cout, groups, dg, H, W = case
    x, wgt, bias, off, mask, _ = _inputs(case, 700, True, F32)
    got = modulated_deform_conv(*_dev(x, off, mask, wgt, bias), 1, 1, 1, 1, dg)
    assert calls == [1]
    _within(got, dco.forward(x, wgt, bias, off, mask, *geo, 1, dg), 2e-5, 'tensor-core route:f32')
    got = modulated_deform_conv(*_dev(x, off, mask, wgt), None, 1, 1, 1, 1, dg)        # bias None: zero bias
    assert calls == [1, 1]
    _within(got, dco.forward(x, wgt, None, off, mask, *geo, 1, dg), 2e-5, 'tensor-core route:f32')
    monkeypatch.setenv('C2M_EXT_DCN_TC', '0')
    modulated_deform_conv(*_dev(x, off, mask, wgt, bias), 1, 1, 1, 1, dg)
    assert calls == [1, 1]


def test_im2col_step_changes_nothing():
    from mmsr.models.archs.dcn import deform_conv
    case = ((3, 3, 1, 1, 1, 1, 1, 1), 4, 6, 6, 3, 2, 9, 8)
    geo, B, C, Cout, groups, dg, H, W = case
    x, wgt, _, off, _, gout = _dev(*_inputs(case, 800, False, F32))
    outs = []
    for step in (1, 2, B, 64):
        leaves = [t.clone().requires_grad_(True) for t in (x, off, wgt)]
        y = deform_conv(leaves[0], leaves[1], leaves[2], 1, 1, 1, groups, dg, step)
        y.backward(gout)
        outs.append((y.detach(), leaves[1].grad, leaves[2].grad))
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1]) and torch.equal(o[2], outs[0][2])
    with pytest.raises(AssertionError, match='im2col step must divide batchsize'):
        deform_conv(x, off, wgt, 1, 1, 1, groups, dg, 3)


def test_reference_style_script():
    """What a caller of the reference package writes: import, build, forward and backward on CUDA tensors."""
    from mmsr.models.archs.dcn import DeformConvPack, ModulatedDeformConvPack
    x = torch.randn(2, 16, 12, 14, device=DEV, requires_grad=True)
    for m in (ModulatedDeformConvPack(16, 32, 3, stride=1, padding=1, deformable_groups=2),
              DeformConvPack(16, 32, 3, stride=1, padding=1, groups=4, deformable_groups=2)):
        m = m.to(DEV)
        y = m(x)
        assert y.shape == (2, 32, 12, 14)
        y.mean().backward()
        assert torch.isfinite(x.grad).all() and torch.isfinite(m.weight.grad).all()


def test_library_errors_raise():
    """A bad argument the Python layer lets through is reported by the library as an exception, not printed."""
    from c2m_b200 import _lib, ops
    x = torch.zeros(1, 6, 5, 5, device=DEV, dtype=F64)
    out = torch.zeros(1, 4, 3, 3, device=DEV, dtype=F64)
    s = ops._shape(x, 4, 3, 3, 1, 1, 0, 0, 1, 1, 1, out)
    rc = _lib.lib().c2m_deform_conv_forward_f64(x.data_ptr(), x.data_ptr(), None, x.data_ptr(), None, 3,
                                                out.data_ptr(), s, ops._stream())
    with pytest.raises(_lib.C2MError, match='divisible by groups'):
        _lib.check(rc, 'c2m_deform_conv_forward_f64')


def _guarded(shape, dtype, pad=4096):
    """A tensor of `shape` in the middle of a buffer whose `pad` elements on each side hold a sentinel."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * pad,), -12345.5, dtype=dtype, device=DEV)
    return buf, buf[pad:pad + n].view(shape), pad


def _guards_intact(buf, pad, what):
    assert bool((buf[:pad] == -12345.5).all()) and bool((buf[-pad:] == -12345.5).all()), f'{what} wrote out of bounds'


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('modulated', [False, True], ids=['v1', 'modulated'])
@pytest.mark.parametrize('case', [CASES[i] for i in (0, 2, 3, 5, 6)], ids=_case_id)
def test_entry_points_write_only_their_outputs_and_forward_is_repeatable(case, modulated, dtype):
    """Each of the c2m_deform_conv_* entry points writes inside its output and nowhere next to it (sentinel guards on
    both sides), and the forward gives the same bits twice (its shared-memory tiles are not raced)."""
    from c2m_b200 import _lib, ops
    geo, B, C, Cout, groups, dg, H, W = case
    kh, kw = geo[:2]
    Ho, Wo = _out_hw(geo, H, W)
    sfx = 'f32' if dtype == F32 else 'f64'
    L = _lib.lib()
    x, wgt, bias, off, mask, gout = _dev(*_inputs(case, 900 + CASES.index(case), modulated, dtype))
    mp = mask.data_ptr() if mask is not None else None
    outs = []
    for _ in range(2):
        buf, out, pad = _guarded((B, Cout, Ho, Wo), dtype)
        s = ops._shape(x, Cout, *geo, dg, out)
        _lib.check(getattr(L, f'c2m_deform_conv_forward_{sfx}')(
            x.data_ptr(), off.data_ptr(), mp, wgt.data_ptr(), bias.data_ptr() if bias is not None else None, groups,
            out.data_ptr(), s, ops._stream()), 'forward')
        _guards_intact(buf, pad, 'forward')
        outs.append(out.clone())
    assert torch.equal(outs[0], outs[1])
    cbuf, cols, pad = _guarded((B, C * kh * kw, Ho * Wo), dtype)
    _lib.check(getattr(L, f'c2m_deform_conv_im2col_{sfx}')(x.data_ptr(), off.data_ptr(), mp, s, cols.data_ptr(),
                                                           ops._stream()), 'im2col')
    _guards_intact(cbuf, pad, 'im2col')
    obuf, goff, pad = _guarded(tuple(off.shape), dtype)
    mbuf, gmask, _ = _guarded(tuple(mask.shape), dtype) if modulated else (None, None, None)
    _lib.check(getattr(L, f'c2m_deform_conv_col2im_coord_{sfx}')(
        cols.data_ptr(), x.data_ptr(), off.data_ptr(), mp, s, goff.data_ptr(),
        gmask.data_ptr() if modulated else None, ops._stream()), 'col2im_coord')
    _guards_intact(obuf, pad, 'col2im_coord grad_offset')
    if modulated:
        _guards_intact(mbuf, pad, 'col2im_coord grad_mask')
    xbuf, gx, pad = _guarded(tuple(x.shape), dtype)
    gx.zero_()
    _lib.check(getattr(L, f'c2m_deform_conv_col2im_{sfx}')(cols.data_ptr(), off.data_ptr(), mp, s, gx.data_ptr(),
                                                           ops._stream()), 'col2im')
    _guards_intact(xbuf, pad, 'col2im')
    assert bool(torch.isfinite(gx).all()) and bool(torch.isfinite(goff).all())
