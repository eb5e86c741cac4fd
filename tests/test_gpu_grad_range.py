"""The tensor-core backwards (ops.conv3x3: dX on conv3x3_wgmma_kernel, dW on conv3x3_wgrad_kernel; ops.dcn_v2_tc:
dcn_dgrad_kernel and dcn_wgrad_kernel) with grad_output across fp32's range, image by image, -m gpu.

grad_output enters the kernels at one power-of-two exponent per image, as x does, so an image's gradients must not
depend on the magnitudes of the other images in the batch.  References and bars are the suite's:
- convolution: the fp64 shifted-slice convolution of tests/golden/conv3x3_ref.py; bar max(1e-5 max|ref|, 2 x the
  error of cuDNN fp32 with TF32 off), as test_gpu_conv3x3_range.py;
- DCN: the fp64 oracle c_oracle.dcn_v2_backward; bar max(1e-5 max|ref|, 2 x the error of `_ext.dcn_v2_backward`), as
  test_gpu_dcn_tc_backward.py.
The per-image gradients (dX, grad_input, grad_offset, grad_mask) are held to the bar image by image, against each
image's own reference; dW and db over the batch.  Every case checks that the tensor-core kernels launched."""
import math
import struct

import pytest
import torch
import torch.nn.functional as F

import conv3x3_ref as R
import seeding

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FLT_MAX = 3.4028234663852886e38
GY = [1e-30, 1e-20, 1e-8, 2.0 ** -19, 1.0, 1e8, 1e20, 1e30]


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def _per_image(scales):
    return torch.tensor(scales, dtype=torch.float32, device=DEV).view(-1, 1, 1, 1)


def _bar_ratio(got, ref, other):
    """error / bar of `got` against the fp64 `ref` over the entries where ref is finite; bar = max(1e-5 max|ref|,
    2 x the error of `other`, a plain fp32 implementation).  inf when an error meets a bar of 0."""
    ref = ref.to(got.device).double()
    fin = torch.isfinite(ref)
    if not bool(fin.any()):
        return 0.0
    r = ref[fin]
    err = float((got[fin].double() - r).abs().max())
    if math.isnan(err):
        return math.inf
    o = other.to(got.device)[fin].double()
    both = torch.isfinite(o)
    err_o = float((o[both] - r[both]).abs().max()) if bool(both.any()) else 0.0
    bar = max(1e-5 * float(r.abs().max()), 2 * err_o)
    return err / bar if bar > 0 else (0.0 if err == 0 else math.inf)


def _worst(got, ref, other, per_image):
    if per_image:
        return max(_bar_ratio(got[i], ref[i], other[i]) for i in range(got.shape[0]))
    return _bar_ratio(got, ref, other)


def _amax_exp(bits, top):
    """Python mirror of amax_exp (umma_conv_common.cuh): top - floor(log2 amax) from amax's fp32 bits, clamped to +-120."""
    if bits == 0:
        return 0
    return max(-120, min(120, top - ((bits >> 23) - 127)))


def _amax_bits(t):
    a = t.detach().abs()
    a = float(a[torch.isfinite(a)].max())
    return struct.unpack('<I', struct.pack('<f', a))[0]


# ---------------------------------------------------------------------------------------------------- convolution
def _conv_inputs(shape, seed, gys=1.0, xs=1.0, ws=1.0):
    """x, w, b, grad_output of one case: x ~ N(0, 1) * xs (a scalar or one scale per image), w at the usual init
    (1 / sqrt(9 Cin)) * ws, b ~ N(0, 0.1^2) * xs, grad_output ~ N(0, 1) * gys (a scalar or one scale per image)."""
    B, cin, cout, H, W = shape
    if isinstance(xs, (list, tuple)):
        x = seeding.randn(seed, (B, cin, H, W)).to(DEV) * _per_image(xs)
        b = seeding.randn(seed + 2, (cout,), 0.1).to(DEV)
    else:
        x = seeding.randn(seed, (B, cin, H, W)).to(DEV) * xs
        b = seeding.randn(seed + 2, (cout,), 0.1).to(DEV) * xs
    w = seeding.randn(seed + 1, (cout, cin, 3, 3), 1.0 / math.sqrt(9 * cin)).to(DEV) * ws
    g = seeding.randn(seed + 3, (B, cout, H, W)).to(DEV)
    gy = g * (_per_image(gys) if isinstance(gys, (list, tuple)) else gys)
    return x, w, b, gy


def _conv_tc(x, w, b, act, gy):
    """(y, dX, dW, db) of ops.conv3x3; asserts that the forward / dX kernel ran twice and the dW kernel once."""
    from c2m_b200 import ops
    ops.profile_enable(True)
    ops.profile_collect('conv3x3')
    ops.profile_collect('conv3x3_wgrad')
    try:
        xr, wr, br = (t.detach().clone().requires_grad_() for t in (x, w, b))
        y = ops.conv3x3(xr, wr, br, act)
        y.backward(gy)
        torch.cuda.synchronize()
        n5, n7 = ops.profile_collect('conv3x3')['launches'], ops.profile_collect('conv3x3_wgrad')['launches']
    finally:
        ops.profile_enable(False)
    assert n5 == 2 and n7 == 1, (n5, n7)
    return y.detach(), xr.grad, wr.grad, br.grad


def _conv_refs(x, w, b, act, y, gy):
    """fp64 reference and cuDNN fp32 of (out, dX, dW, db), the backward through the mask of the op's own output y."""
    g = gy if act is None else torch.where(y > 0, gy, 0. if act == 'relu' else gy * 0.1)
    act_f = (lambda t: t) if act is None else (F.relu if act == 'relu' else (lambda t: F.leaky_relu(t, 0.1)))
    ref = (act_f(R.conv3x3_forward(x, w, b)),) + R.conv3x3_grads(x, w, g)
    c32 = (act_f(F.conv2d(x, w, b, 1, 1)), torch.nn.grad.conv2d_input(x.shape, w, g, 1, 1),
           torch.nn.grad.conv2d_weight(x, w.shape, g, 1, 1), g.sum((0, 2, 3)))
    return ref, c32


CONV_NAMES = ('out', 'dX', 'dW', 'db')


def _conv_ratios(got, ref, c32):
    """{name: worst error / bar}: out and dX image by image, dW and db over the batch."""
    return {n: _worst(g, r, c, n in ('out', 'dX')) for n, g, r, c in zip(CONV_NAMES, got, ref, c32)}


# (B, Cin, Cout, H, W): the stage-3 64 -> 64 layer at 40 x 40, a map ragged in rows and columns, and conv_first's 3 input
# channels on the smallest map
CONV_SHAPES = [(2, 64, 64, 40, 40), (2, 48, 40, 130, 70), (3, 3, 48, 19, 11)]
ACTS = [None, 'relu', 'lrelu']


@pytest.mark.parametrize('gy', GY)
def test_conv_uniform_grad_scale(gy):
    """grad_output ~ N(0, 1) * s for s from 1e-30 to 1e30 on each shape: every output finite and within the bar."""
    bad = []
    for si, shape in enumerate(CONV_SHAPES):
        act = ACTS[(si + GY.index(gy)) % 3]
        x, w, b, g = _conv_inputs(shape, 100 + si, gy)
        got = _conv_tc(x, w, b, act, g)
        ref, c32 = _conv_refs(x, w, b, act, got[0], g)
        r = _conv_ratios(got, ref, c32)
        print(f'{shape} {act} gy~{gy:g}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
        bad += [(shape, n) for n, t in zip(CONV_NAMES, got) if not bool(torch.isfinite(t).all())]
        bad += [(shape, r)] if max(r.values()) > 1.0 else []
    assert not bad, bad


MIXED = {'1e5': ([1.0, 1e-5, 1e5], 1.0), '2^40': ([1.0, 2.0 ** -40, 2.0 ** 40], 1.0),
         'x_opposite': ([1.0, 1e-5, 1e5], [1.0, 1e5, 1e-5])}


@pytest.mark.parametrize('mix', MIXED)
def test_conv_mixed_grad_scale_batch(mix):
    """grad_output of magnitudes 2^-19 x {1, 1e-5, 1e5} or {1, 2^-40, 2^40} in one batch (and once with x scaled per
    image the opposite way, so that x * grad_output stays O(1) per image): dX within the bar of each image's own
    reference, out / dW / db as usual."""
    gys, xs = MIXED[mix]
    x, w, b, gy = _conv_inputs((3, 64, 64, 40, 40), 200, [s * 2.0 ** -19 for s in gys], xs)
    got = _conv_tc(x, w, b, 'lrelu', gy)
    ref, c32 = _conv_refs(x, w, b, 'lrelu', got[0], gy)
    r = _conv_ratios(got, ref, c32)
    print(f'mixed {mix}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    assert max(r.values()) <= 1.0, r


def test_conv_grad_scale_per_image_exact_and_independent():
    """Image 1's grad_output times 2^-40 or 2^40: image 1's dX exactly that factor times, image 0's the same bits.  In a
    batch of grad_output magnitudes {1, 1e-5, 1e5}, each image's dX equals, bit for bit, the same image run alone."""
    x, w, b, gy = _conv_inputs((3, 64, 64, 40, 40), 300, 2.0 ** -19)
    _, dx0, _, _ = _conv_tc(x, w, b, 'relu', gy)
    for k in (-40, 40):
        g = gy.clone()
        g[1] *= 2.0 ** k
        _, dx, _, _ = _conv_tc(x, w, b, 'relu', g)
        assert torch.equal(dx[1], dx0[1] * 2.0 ** k), k
        assert torch.equal(dx[0], dx0[0]) and torch.equal(dx[2], dx0[2]), k
    g = gy * _per_image([1.0, 1e-5, 1e5])
    _, dx, _, _ = _conv_tc(x, w, b, 'relu', g)
    for i in range(3):
        _, dxi, _, _ = _conv_tc(x[i:i + 1], w, b, 'relu', g[i:i + 1])
        assert torch.equal(dxi, dx[i:i + 1]), i


@pytest.mark.parametrize('kind', ['zero', 'nan', 'inf', '-inf'])
def test_conv_degenerate_grad_image(kind):
    """Image 1's grad_output all zero: its dX exactly 0, image 0's dX the same bits as image 0 run alone.  All NaN /
    +-Inf: the finiteness patterns of dX, dW and db equal the reference's and image 0's dX is within its bar."""
    x, w, b, gy = _conv_inputs((2, 40, 24, 21, 13), 400, 2.0 ** -19)
    gy[1] = {'zero': 0.0, 'nan': float('nan'), 'inf': float('inf'), '-inf': float('-inf')}[kind]
    got = _conv_tc(x, w, b, None, gy)
    if kind == 'zero':
        assert bool((got[1][1] == 0).all())
        _, dx_alone, _, _ = _conv_tc(x[:1], w, b, None, gy[:1])
        assert torch.equal(got[1][:1], dx_alone)
        return
    ref, c32 = _conv_refs(x, w, b, None, got[0], gy)
    for n, g, r in zip(CONV_NAMES[1:], got[1:], ref[1:]):
        assert bool((~torch.isfinite(r)).any()), n
        assert torch.equal(torch.isfinite(g), torch.isfinite(r)), n
    assert _bar_ratio(got[1][0], ref[1][0], c32[1][0]) <= 1.0


def _check_bottom(scale_name, t_amax, w):
    """Asserts the case is at the bottom of the normal range: 2^-(s_b + sw) (input exponent from t's amax, weight
    exponent 13 - floor(log2 max|w|) as wpack_scale) is below fp32's smallest subnormal."""
    sw = 13 - ((_amax_bits(w) >> 23) - 127)
    for i in range(t_amax.shape[0]):
        s_b = _amax_exp(_amax_bits(t_amax[i]), 14)
        assert s_b + sw > 149, (scale_name, i, s_b, sw)


@pytest.mark.parametrize('which', ['out', 'dX'])
def test_conv_bottom_of_normal_range(which):
    """x (for out) or grad_output (for dX) ~ 2^-100 N(0, 1) and w at 2^-22 times the usual init, bias 0: 2^-(s_b + sw)
    is not an fp32 number, but the true output (~2^-120) is a normal float; every result within the bar, and that
    output also within 1e-5 max|ref| of each image alone (cuDNN's own products are fp32 subnormals here, which makes
    the suite's bar loose)."""
    shape = (2, 64, 64, 40, 40)
    tiny = 2.0 ** -100
    x, w, b, gy = _conv_inputs(shape, 500, tiny if which == 'dX' else 2.0 ** -19, tiny if which == 'out' else 1.0,
                               2.0 ** -22)
    b = torch.zeros_like(b)
    _check_bottom(which, x if which == 'out' else gy, w)
    got = _conv_tc(x, w, b, None, gy)
    ref, c32 = _conv_refs(x, w, b, None, got[0], gy)
    k = CONV_NAMES.index(which)
    m = float(ref[k].abs().max())
    assert 2.0 ** -121 <= m <= 2.0 ** -110, m
    r = _conv_ratios(got, ref, c32)
    strict = max(float((got[k][i].double() - ref[k][i]).abs().max() / (1e-5 * ref[k][i].abs().max()))
                 for i in range(shape[0]))
    print(f'bottom {which}: max |ref| 2^{math.log2(m):.1f} ' + ' '.join(f'{n} {v:.3f}' for n, v in r.items()) +
          f' {which} error / 1e-5 max|ref| {strict:.3f}')
    assert max(r.values()) <= 1.0, r
    assert strict <= 1.0, strict


CROSS = [(1e30, 1e-30), (1e-30, 1e30), (1e20, 1e-25)]


def _normal_range(ref):
    m = float(ref.double().abs().max())
    return m <= FLT_MAX and m * 1e-5 >= 2.0 ** -126


@pytest.mark.parametrize('xs,gys', CROSS, ids=[f'x{a:g}_gy{g:g}' for a, g in CROSS])
def test_conv_cross_range(xs, gys):
    """x and grad_output at opposite ends of fp32's range: dW, db and dX within the bar wherever the fp64 result is a
    normal float, so that no partial sum, workspace slot or flush product leaves fp32's range once the per-image
    exponents are combined."""
    x, w, b, gy = _conv_inputs((2, 64, 64, 40, 40), 600, gys, xs)
    got = _conv_tc(x, w, b, 'lrelu', gy)
    ref, c32 = _conv_refs(x, w, b, 'lrelu', got[0], gy)
    r = {n: v for n, v, rf in zip(CONV_NAMES, _conv_ratios(got, ref, c32).values(), ref) if _normal_range(rf)}
    print(f'cross x~{xs:g} gy~{gys:g}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    assert {'dX', 'dW', 'db'} <= set(r), r
    assert max(r.values()) <= 1.0, r


# ------------------------------------------------------------------------------------------------------------- DCN
def _dcn_inputs(case, seed, gys=1.0, xs=1.0, ws=1.0):
    """x ~ N(0, 1) * xs, offsets ~ N(0, 2^2), sigmoid mask, w at 1 / sqrt(9 C) * ws, grad_output ~ N(0, 1) * gys (xs and
    gys: a scalar or one scale per image)."""
    B, C, cout, H, W, dg = case
    sc = lambda s: _per_image(s) if isinstance(s, (list, tuple)) else s  # noqa: E731
    x = seeding.randn(seed, (B, C, H, W)).to(DEV) * sc(xs)
    off = seeding.randn(seed + 1, (B, 18 * dg, H, W), 2.0).to(DEV)
    mask = torch.sigmoid(seeding.randn(seed + 2, (B, dg * 9, H, W))).to(DEV)
    w = seeding.randn(seed + 3, (cout, C, 3, 3), (9 * C) ** -0.5).to(DEV) * ws
    b = seeding.randn(seed + 4, (cout,), 0.1).to(DEV)
    gy = seeding.randn(seed + 5, (B, cout, H, W)).to(DEV) * sc(gys)
    return x, off, mask, w, b, gy, dg


DCN_NAMES = ('grad_input', 'grad_offset', 'grad_mask', 'grad_weight', 'grad_bias')


def _dcn_tc(x, off, mask, w, b, gy, dg):
    """(grad_input, grad_offset, grad_mask, grad_weight, grad_bias) of ops.dcn_v2_tc; asserts that dcn_dgrad_kernel and
    dcn_wgrad_kernel each launched once."""
    from c2m_b200 import ops
    ops.profile_enable(True)
    ops.profile_collect('dcn_dgrad')
    ops.profile_collect('dcn_wgrad')
    try:
        leaves = [t.detach().clone().requires_grad_() for t in (x, off, mask, w, b)]
        ops.dcn_v2_tc(*leaves, dg).backward(gy)
        torch.cuda.synchronize()
        nd, nw = ops.profile_collect('dcn_dgrad')['launches'], ops.profile_collect('dcn_wgrad')['launches']
    finally:
        ops.profile_enable(False)
    assert nd == 1 and nw == 1, (nd, nw)
    return tuple(t.grad for t in leaves)


def _dcn_refs(x, off, mask, w, b, gy, dg):
    """fp64 oracle and `_ext` (fp32 CUDA cores, no operand scaling) of the five gradients."""
    from c2m_b200 import ops
    from oracle import c_oracle
    ref = c_oracle.dcn_v2_backward(x.cpu().double(), w.cpu().double(), b.cpu().double(), off.cpu().double(),
                                   mask.cpu().double(), gy.cpu().double(), dg=dg)
    ext = ops.dcn_v2_backward(x, w, b, off, mask, gy, 3, 3, 1, 1, 1, 1, 1, 1, dg)
    return ref, ext


def _dcn_ratios(got, ref, ext, only=None):
    return {n: _worst(g, r, e, i < 3) for i, (n, g, r, e) in enumerate(zip(DCN_NAMES, got, ref, ext))
            if only is None or n in only}


# (B, C, Cout, H, W, dg): a stage-3 shape on a small map, Cout partial in the wgrad slice, and a column count C * 9 that
# is not a multiple of dcn_dgrad_kernel's chunk width (a partial last chunk)
DCN_SHAPES = [(2, 64, 64, 24, 16, 8), (3, 64, 40, 33, 27, 4), (2, 32, 32, 19, 11, 1)]


@pytest.mark.parametrize('gy', GY)
def test_dcn_uniform_grad_scale(gy):
    """grad_output ~ N(0, 1) * s for s from 1e-30 to 1e30 on each shape: every gradient finite and within the bar."""
    bad = []
    for si, case in enumerate(DCN_SHAPES):
        args = _dcn_inputs(case, 700 + 10 * si, gy)
        got = _dcn_tc(*args)
        ref, ext = _dcn_refs(*args)
        r = _dcn_ratios(got, ref, ext)
        print(f'{case} gy~{gy:g}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
        bad += [(case, n) for n, t in zip(DCN_NAMES, got) if not bool(torch.isfinite(t).all())]
        bad += [(case, r)] if max(r.values()) > 1.0 else []
    assert not bad, bad


@pytest.mark.parametrize('mix', MIXED)
def test_dcn_mixed_grad_scale_batch(mix):
    """The convolution's mixed batches on the DCN: grad_input, grad_offset and grad_mask within the bar of each image's
    own reference, grad_weight and grad_bias over the batch."""
    gys, xs = MIXED[mix]
    args = _dcn_inputs((3, 64, 64, 24, 16, 8), 800, [s * 2.0 ** -19 for s in gys], xs)
    got = _dcn_tc(*args)
    ref, ext = _dcn_refs(*args)
    r = _dcn_ratios(got, ref, ext)
    print(f'mixed {mix}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    assert max(r.values()) <= 1.0, r


def test_dcn_grad_scale_per_image_exact_and_independent():
    """Image 1's grad_output times 2^-40 or 2^40: image 1's grad_offset and grad_mask exactly that factor times, image
    0's the same bits (grad_input is summed with atomics: held to the bar).  In a batch of grad_output magnitudes
    {1, 1e-5, 1e5}, each image's grad_offset and grad_mask equal, bit for bit, the same image run alone."""
    x, off, mask, w, b, gy, dg = _dcn_inputs((3, 64, 64, 24, 16, 8), 900, 2.0 ** -19)
    g0 = _dcn_tc(x, off, mask, w, b, gy, dg)
    for k in (-40, 40):
        g = gy.clone()
        g[1] *= 2.0 ** k
        gk = _dcn_tc(x, off, mask, w, b, g, dg)
        for j in (1, 2):
            assert torch.equal(gk[j][1], g0[j][1] * 2.0 ** k), (k, DCN_NAMES[j])
            assert torch.equal(gk[j][0], g0[j][0]) and torch.equal(gk[j][2], g0[j][2]), (k, DCN_NAMES[j])
        ref, ext = _dcn_refs(x, off, mask, w, b, g, dg)
        assert _worst(gk[0], ref[0], ext[0], True) <= 1.0, k
    g = gy * _per_image([1.0, 1e-5, 1e5])
    gm = _dcn_tc(x, off, mask, w, b, g, dg)
    for i in range(3):
        s = slice(i, i + 1)
        gi = _dcn_tc(x[s], off[s], mask[s], w, b, g[s], dg)
        assert torch.equal(gi[1], gm[1][s]) and torch.equal(gi[2], gm[2][s]), i


@pytest.mark.parametrize('kind', ['zero', 'nan', 'inf', '-inf'])
def test_dcn_degenerate_grad_image(kind):
    """Image 1's grad_output all zero: its grad_input, grad_offset and grad_mask exactly 0, image 0's grad_offset and
    grad_mask the same bits as image 0 run alone.  All NaN / +-Inf: the finiteness pattern of every gradient equals the
    oracle's and image 0's per-image gradients are within their bar."""
    x, off, mask, w, b, gy, dg = _dcn_inputs((2, 64, 64, 19, 11, 8), 1000, 2.0 ** -19)
    gy[1] = {'zero': 0.0, 'nan': float('nan'), 'inf': float('inf'), '-inf': float('-inf')}[kind]
    got = _dcn_tc(x, off, mask, w, b, gy, dg)
    if kind == 'zero':
        for j in range(3):
            assert bool((got[j][1] == 0).all()), DCN_NAMES[j]
        alone = _dcn_tc(x[:1], off[:1], mask[:1], w, b, gy[:1], dg)
        assert torch.equal(alone[1], got[1][:1]) and torch.equal(alone[2], got[2][:1])
        return
    ref, ext = _dcn_refs(x, off, mask, w, b, gy, dg)
    for n, g, r in zip(DCN_NAMES, got, ref):
        assert torch.equal(torch.isfinite(g).cpu(), torch.isfinite(r)), n
    for j in range(3):
        assert _bar_ratio(got[j][0], ref[j][0], ext[j][0]) <= 1.0, DCN_NAMES[j]


def test_dcn_bottom_of_normal_range():
    """grad_output ~ 2^-100 N(0, 1) and w at 2^-22 times the usual init, the convolution's dX case: every gradient
    within the bar."""
    args = _dcn_inputs((2, 64, 64, 24, 16, 8), 1100, 2.0 ** -100, 1.0, 2.0 ** -22)
    got = _dcn_tc(*args)
    ref, ext = _dcn_refs(*args)
    m = float(ref[0].double().abs().max())
    assert 2.0 ** -124 <= m <= 2.0 ** -110, m
    r = _dcn_ratios(got, ref, ext)
    print(f'bottom: max |grad_input| 2^{math.log2(m):.1f} ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('xs,gys', CROSS, ids=[f'x{a:g}_gy{g:g}' for a, g in CROSS])
def test_dcn_cross_range(xs, gys):
    """x and grad_output at opposite ends of fp32's range: every gradient whose fp64 result is a normal float within
    the bar (gcol, the gathered columns and the flushes stay inside fp32's range)."""
    args = _dcn_inputs((2, 64, 64, 24, 16, 8), 1200, gys, xs)
    got = _dcn_tc(*args)
    ref, ext = _dcn_refs(*args)
    keep = {n for n, r in zip(DCN_NAMES, ref) if _normal_range(r)}
    r = _dcn_ratios(got, ref, ext, keep)
    print(f'cross x~{xs:g} gy~{gys:g}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    assert {'grad_input', 'grad_weight'} <= set(r), r
    assert max(r.values()) <= 1.0, r


# ------------------------------------------------------------------------------------------------------ end to end
def test_restoration_net_per_image_loss_weights():
    """RestorationNet(64, 16, 8), B = 2, set up as test_gpu_dcn_tc_backward's training step, with the LR input
    requiring grad.  One forward, two backwards: of l0 + 2^-30 l1 and of l0 + l1 (l: the per-image L1 losses).  Image
    1's input gradient from the first, times 2^30, matches the second, and image 0's matches too, each within 1e-6
    relative L2: a small loss weight on one image does not cost that image's gradient its precision.  Measured on an
    H100: 1.3e-7 for image 1 and 1.2e-7 for image 0 (the order of grad_input's atomic sums); 2.2e-3 for image 1 with one
    grad_output exponent for the whole batch."""
    from c2m_b200 import ops
    from mmsr.models.archs.corres_generation_arch import CorrespondenceGenerationArch
    from mmsr.models.archs.ref_restoration_arch import RestorationNet
    net_map = CorrespondenceGenerationArch(3, 1, ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19')
    net_map.load_state_dict(seeding.seeded_state_dict(seeding.spec_net_map(), 12))
    net_map.to(DEV).eval()
    net_g = RestorationNet(64, 16, 8)
    net_g.load_state_dict(seeding.seeded_state_dict(seeding.spec_restoration_net(), 13))
    net_g.to(DEV).train()
    B, lr = 2, 40
    hr = seeding.structured_image(31, B, 4 * lr).to(DEV)
    x = F.interpolate(hr, scale_factor=0.25, mode='bicubic', align_corners=False).clamp(0, 1)
    f1 = seeding.randn(32, (B, 256, lr, lr)).to(DEV)
    f2 = (f1 + seeding.randn(33, (B, 256, lr, lr), 0.1).to(DEV)).roll(3, 3)
    img_ref = seeding.structured_image(34, B, 4 * lr).to(DEV)
    with torch.no_grad():
        pre, feats = net_map({'dense_features1': f1, 'dense_features2': f2}, img_ref)
    x = x.detach().requires_grad_()
    ops.profile_enable(True)
    for k in ('conv3x3', 'conv3x3_wgrad', 'dcn_dgrad', 'dcn_wgrad'):
        ops.profile_collect(k)
    try:
        l = (net_g(x, pre, feats) - hr).abs().mean((1, 2, 3))
        g_small, = torch.autograd.grad(l[0] + 2.0 ** -30 * l[1], x, retain_graph=True)
        g_even, = torch.autograd.grad(l[0] + l[1], x)
        torch.cuda.synchronize()
        n = {k: ops.profile_collect(k)['launches'] for k in ('conv3x3_wgrad', 'dcn_dgrad', 'dcn_wgrad')}
    finally:
        ops.profile_enable(False)
    assert n['conv3x3_wgrad'] > 0 and n['dcn_dgrad'] == 6 and n['dcn_wgrad'] == 6, n

    def rel(a, b):
        return float((a.double() - b.double()).norm() / b.double().norm())
    d1, d0 = rel(g_small[1] * 2.0 ** 30, g_even[1]), rel(g_small[0], g_even[0])
    print(f'relative L2: image 1 (loss weight 2^-30) {d1:.3e}, image 0 {d0:.3e}')
    assert d1 <= 1e-6 and d0 <= 1e-6, (d1, d0)
