"""The tensor-core 3x3 convolution (ops.conv3x3: forward and dX on conv3x3_wgmma_kernel, dW on conv3x3_wgrad_kernel)
across fp32's range and with non-finite inputs, -m gpu.

Reference: the fp64 shifted-slice convolution of tests/golden/conv3x3_ref.py (run on the GPU in fp64; its agreement
with torch's fp64 functions, values and finiteness, is checked on the CPU by test_conv3x3_nonfinite_reference.py).
Bar, per gradient: max(1e-5 max|ref|, 2 x the error of cuDNN fp32 with TF32 off on the same case), as
test_gpu_conv3x3_backward.py; the forward is held to it image by image against each image's own output scale.  The
activation's mask is the op's own forward output.  Every case checks that both kernels launched."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import conv3x3_ref as R
import seeding

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def _inputs(shape, seed, xs=1.0, ws=None):
    B, cin, cout, H, W = shape
    x = seeding.randn(seed, (B, cin, H, W), 1.0).to(DEV) * xs
    w = seeding.randn(seed + 1, (cout, cin, 3, 3), ws or 1.0 / math.sqrt(9 * cin)).to(DEV)
    b = seeding.randn(seed + 2, (cout,), 0.1).to(DEV) * xs
    gy = seeding.randn(seed + 3, (B, cout, H, W), 2.0 ** -19).to(DEV)
    return x, w, b, gy


def _tc(x, w, b, act, gy):
    """(y, dX, dW, db) of ops.conv3x3, and asserts that the forward / dX kernel and the dW kernel both launched."""
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


def _masked(y, gy, act):
    if act == 'relu':
        return torch.where(y > 0, gy, 0.)
    if act == 'lrelu':
        return torch.where(y > 0, gy, gy * 0.1)
    return gy


def _act(y, act):
    return F.relu(y) if act == 'relu' else F.leaky_relu(y, 0.1) if act == 'lrelu' else y


def _refs(x, w, b, act, y, gy):
    """fp64 reference and cuDNN fp32 of (out, dX, dW, db); the backward for the mask of the op's own output y."""
    g = _masked(y, gy, act)
    ref = (_act(R.conv3x3_forward(x, w, b), act),) + R.conv3x3_grads(x, w, g)
    c32 = (_act(F.conv2d(x, w, b, 1, 1), act), torch.nn.grad.conv2d_input(x.shape, w, g, 1, 1),
           torch.nn.grad.conv2d_weight(x, w.shape, g, 1, 1), g.sum((0, 2, 3)))
    return ref, c32


def _ratio(got, ref, c32):
    """error / bar over the entries where the reference is finite (inf when a bar of 0 meets an error)."""
    fin = torch.isfinite(ref)
    if not bool(fin.any()):
        return 0.0
    r = ref[fin]
    err = float((got[fin].double() - r).abs().max())
    if math.isnan(err):
        return math.inf
    both = fin & torch.isfinite(c32)
    err32 = float((c32[both].double() - ref[both]).abs().max()) if bool(both.any()) else 0.0
    bar = max(1e-5 * float(r.abs().max()), 2 * err32)
    return err / bar if bar > 0 else (0.0 if err == 0 else math.inf)


def _ratios(got, ref, c32, per_image_fwd=True, per_image_dx=False):
    """{name: worst error / bar}: out (and dX when asked) image by image, the rest over the batch."""
    out = {}
    for i, name in enumerate(('out', 'dX', 'dW', 'db')):
        if (name == 'out' and per_image_fwd) or (name == 'dX' and per_image_dx):
            out[name] = max(_ratio(got[i][k], ref[i][k], c32[i][k]) for k in range(got[i].shape[0]))
        else:
            out[name] = _ratio(got[i], ref[i], c32[i])
    return out


# (B, Cin, Cout, H, W): the stage-3 64 -> 64 and 320 -> 256 (two Cout slices) layers at 40 x 40, then maps that are
# not a multiple of the 16 x 8 tile in rows, columns or both
SHAPES = [(2, 64, 64, 40, 40), (2, 320, 256, 40, 40), (2, 48, 40, 130, 70), (3, 3, 48, 19, 11), (2, 40, 72, 19, 11)]
SCALES = [1e-30, 1e-6, 1e-3, 1.0, 1e4, 1e30]
ACTS = [None, 'relu', 'lrelu']


@pytest.mark.parametrize('scale', SCALES)
@pytest.mark.parametrize('si', range(len(SHAPES)), ids=['x'.join(map(str, s)) for s in SHAPES])
def test_input_scale_vs_fp64(si, scale):
    """x and bias at scale s: out, dX, dW and db within the bar at every s from 1e-30 to 1e30."""
    shape = SHAPES[si]
    act = ACTS[(si + SCALES.index(scale)) % 3]
    x, w, b, gy = _inputs(shape, 1000 + si, scale)
    got = _tc(x, w, b, act, gy)
    ref, c32 = _refs(x, w, b, act, got[0], gy)
    r = _ratios(got, ref, c32)
    print(f'{shape} {act} x~{scale:g}: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    for name, t in zip(('out', 'dX', 'dW', 'db'), got):
        assert bool(torch.isfinite(t).all()), name
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('act', ACTS)
def test_power_of_two_scaling_is_exact(act):
    """x and b times 2^k: out and dW exactly 2^k times, dX and db the same bits; w and b times 2^k: out and dX exactly
    2^k times, dW and db the same bits."""
    shape = (2, 64, 64, 40, 40) if act != 'relu' else (3, 3, 48, 19, 11)
    x, w, b, gy = _inputs(shape, 2000)
    y0, dx0, dw0, db0 = _tc(x, w, b, act, gy)
    bad = []
    for k in (-11, 11, 24, 60):
        s = 2.0 ** k
        y, dx, dw, db = _tc(x * s, w, b * s, act, gy)
        for n, got, want in (('out', y, y0 * s), ('dW', dw, dw0 * s), ('dX', dx, dx0), ('db', db, db0)):
            if not torch.equal(got, want):
                bad.append(('x', k, n))
    for k in (-100, -24, 24, 100):
        s = 2.0 ** k
        y, dx, dw, db = _tc(x, w * s, b * s, act, gy)
        for n, got, want in (('out', y, y0 * s), ('dX', dx, dx0 * s), ('dW', dw, dw0), ('db', db, db0)):
            if not torch.equal(got, want):
                bad.append(('w', k, n))
    assert not bad, bad


@pytest.mark.parametrize('shape', [(3, 64, 64, 40, 40), (3, 3, 48, 19, 11)], ids=['64x64_40x40', '3x48_19x11'])
def test_mixed_scale_batch(shape):
    """Images of magnitude 1, 1e-5 and 1e5 in one batch: out and dX image by image against each image's own scale,
    dW and db over the batch; each image's forward equals, bit for bit, the same image run alone."""
    from c2m_b200 import ops
    x, w, b, gy = _inputs(shape, 3000)
    x = x * torch.tensor([1.0, 1e-5, 1e5], device=DEV).view(-1, 1, 1, 1)
    got = _tc(x, w, b, 'lrelu', gy)
    ref, c32 = _refs(x, w, b, 'lrelu', got[0], gy)
    r = _ratios(got, ref, c32, per_image_dx=True)
    print(f'{shape} mixed: ' + ' '.join(f'{k} {v:.3f}' for k, v in r.items()))
    assert max(r.values()) <= 1.0, r
    with torch.no_grad():
        for i in range(3):
            assert torch.equal(ops.conv3x3(x[i:i + 1], w, b, 'lrelu'), got[0][i:i + 1]), i


def _pixels(H, W):
    return [(0, 0), (H - 1, W - 1), (H - 1, W // 2), (H // 2, W - 1), (H // 3, W // 3)]


def _pattern_and_values(got, ref, c32, what):
    """Mismatches of the finiteness pattern, then of the finite entries against the bar."""
    bad = []
    for name, g, r, c in zip(('out', 'dX', 'dW', 'db'), got, ref, c32):
        if not torch.equal(torch.isfinite(g), torch.isfinite(r)):
            n = int((torch.isfinite(g) != torch.isfinite(r)).sum())
            bad.append((what, name, f'{n} entries differ in finiteness'))
        elif _ratio(g, r, c) > 1.0:
            bad.append((what, name, f'error / bar {_ratio(g, r, c):.3g}'))
    return bad


@pytest.mark.parametrize('bad', ['nan', 'inf', '-inf'])
@pytest.mark.parametrize('hw', [(21, 13), (40, 40), (19, 11), (32, 16)], ids=['21x13', '40x40', '19x11', '32x16'])
def test_nonfinite_x_pattern_equals_reference(hw, bad):
    """One NaN / +-Inf in x (image 1, channel 5) at a corner, the middle of the last row or column, or an interior
    pixel, on maps ragged in rows, columns, both, and a multiple of the tile: the finiteness patterns of out, dX, dW and
    db equal the reference's (in particular dW keeps the taps finite that only pixels outside the map would pair with
    the value), and the finite entries meet the bar."""
    H, W = hw
    x0, w, b, gy = _inputs((2, 40, 24, H, W), 4000)
    mism = []
    for (py, px) in _pixels(H, W):
        x = x0.clone()
        x[1, 5, py, px] = float(bad)
        got = _tc(x, w, b, None, gy)
        ref, c32 = _refs(x, w, b, None, got[0], gy)
        mism += _pattern_and_values(got, ref, c32, (py, px))
    assert not mism, mism


@pytest.mark.parametrize('wscale', [1.0, 2.0 ** 10], ids=['w1', 'w2^10'])
@pytest.mark.parametrize('bad', ['nan', 'inf', '-inf'])
def test_nonfinite_weight(bad, wscale):
    """One NaN / +-Inf weight among weights of magnitude ~1 or ~2^10.  At the centre tap: the patterns of out and dX
    equal the reference's and every finite entry meets the bar (dW and db do not depend on the weights).  At a corner
    tap: the pattern of out (the reference multiplies the zero padding by the weight, as F.conv2d does).  The input
    gradient is not compared there: it runs the forward kernel on the zero-padded grad_output, so the padding meets the
    rotated weight at the border, where the scatter-form reference (torch.nn.grad.conv2d_input) has no term."""
    H, W = 21, 13
    x, w0, b, gy = _inputs((2, 40, 24, H, W), 5000, ws=wscale)
    mism = []
    for ky, kx in ((1, 1), (0, 0)):
        w = w0.clone()
        w[7, 11, ky, kx] = float(bad)
        got = _tc(x, w, b, None, gy)
        ref, c32 = _refs(x, w, b, None, got[0], gy)
        if (ky, kx) == (1, 1):
            mism += _pattern_and_values(got, ref, c32, (ky, kx))
        else:
            mism += _pattern_and_values(got[:1], ref[:1], c32[:1], (ky, kx))
    assert not mism, mism


def _dcn_case(seed, wscale):
    B, C, cout, H, W, dg = 2, 64, 64, 19, 11, 8
    x = seeding.randn(seed, (B, C, H, W)).to(DEV)
    off = seeding.randn(seed + 1, (B, 18 * dg, H, W), 2.0).to(DEV)
    mask = torch.sigmoid(seeding.randn(seed + 2, (B, dg * 9, H, W))).to(DEV)
    w = seeding.randn(seed + 3, (cout, C, 3, 3), wscale).to(DEV)
    b = seeding.randn(seed + 4, (cout,), 0.1).to(DEV)
    gy = seeding.randn(seed + 5, (B, cout, H, W), 2.0 ** -19).to(DEV)
    return x, off, mask, w, b, gy, dg


@pytest.mark.parametrize('bad', ['nan', 'inf'])
def test_nonfinite_weight_dcn_packs(bad):
    """The tensor-core DCN's forward pack (`_ext.dcn_v2_forward`) and dgrad pack (ops.dcn_v2_tc backward) share the
    weight header: one non-finite weight among weights of magnitude ~2^10 leaves every other output channel of the
    forward and every other input channel of grad_input finite and within the bar of the fp64 oracle."""
    from c2m_b200 import ops
    from oracle import c_oracle
    x, off, mask, w, b, gy, dg = _dcn_case(6000, 2.0 ** 10)
    co, ci = 9, 21
    w[co, ci, 0, 2] = float(bad)
    ops.profile_enable(True)
    ops.profile_collect('dcn')
    ops.profile_collect('dcn_dgrad')
    try:
        y = ops.dcn_v2_forward(x, w, b, off, mask, 3, 3, 1, 1, 1, 1, 1, 1, dg)
        xr = x.clone().requires_grad_()
        ops.dcn_v2_tc(xr, off, mask, w, b, dg).backward(gy)
        torch.cuda.synchronize()
        n_fwd, n_dgrad = ops.profile_collect('dcn')['launches'], ops.profile_collect('dcn_dgrad')['launches']
    finally:
        ops.profile_enable(False)
    assert n_fwd == 2 and n_dgrad == 1, (n_fwd, n_dgrad)
    wf = w.clone()
    wf[co, ci, 0, 2] = 0.0
    want_y = c_oracle.dcn_v2_forward(x.cpu(), wf.cpu(), b.cpu(), off.cpu(), mask.cpu(), dg=dg).double()
    want_gx = c_oracle.dcn_v2_backward(x.cpu().double(), wf.cpu().double(), b.cpu().double(), off.cpu().double(),
                                       mask.cpu().double(), gy.cpu().double(), dg=dg)[0]
    keep_o = torch.arange(w.shape[0]) != co
    keep_i = torch.arange(w.shape[1]) != ci
    for name, got, want, keep in (('out', y, want_y, keep_o), ('grad_input', xr.grad, want_gx, keep_i)):
        g, r = got.cpu()[:, keep].double(), want[:, keep]
        assert bool(torch.isfinite(g).all()), name
        err = float((g - r).abs().max())
        assert err <= 1e-5 * float(r.abs().max()), (name, err, float(r.abs().max()))
    assert not bool(torch.isfinite(y[:, co]).all())


def test_no_host_synchronisation():
    """Forward and backward enqueue without a host synchronisation (the exponents stay on the device)."""
    from c2m_b200 import ops
    x, w, b, gy = _inputs((2, 40, 72, 19, 11), 7000, 1e-20)
    xr, wr, br = (t.clone().requires_grad_() for t in (x, w, b))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        y = ops.conv3x3(xr, wr, br, 'relu')
        y.backward(gy)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    ref, c32 = _refs(x, w, b, 'relu', y.detach(), gy)
    r = _ratios((y.detach(), xr.grad, wr.grad, br.grad), ref, c32)
    assert max(r.values()) <= 1.0, r


GUARD = 4096


def _guarded(n, dtype):
    buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=dtype, device=DEV)
    if dtype != torch.float32:
        buf.fill_(-12345)
    return buf


def _guards_intact(buf, n):
    edge = torch.cat([buf[:GUARD], buf[GUARD + n:]])
    return bool(edge.isnan().all()) if buf.dtype == torch.float32 else bool((edge == -12345).all())


@pytest.mark.parametrize('shape', [(2, 40, 72, 19, 11), (3, 3, 48, 21, 13)], ids=['40to72_19x11', '3to48_21x13'])
def test_operand_and_kernels_write_inside_their_buffers_per_image_grad(shape):
    """c2m_conv3x3_operand_f32 (the PSA operand and its per-image amax), the forward with those exponents (fp32 output)
    and c2m_conv3x3_wgrad_scaled with them (dW, workspace) write only inside their buffers, between sentinel guards, and give
    the op's results bit for bit."""
    from c2m_b200 import _lib, ops
    B, cin, cout, H, W = shape
    x, w, b, gy = _inputs(shape, 8000, 1e-7)
    y_op, _, dw_op, _ = _tc(x, w, b, None, gy)
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    c8i = (cin + 7) // 8
    npsa = B * c8i * H * W * 8
    xhi, xlo, amax = _guarded(npsa, torch.float16), _guarded(npsa, torch.float16), _guarded(B, torch.float32)
    _lib.check(L.c2m_conv3x3_operand_f32(x.data_ptr(), B, cin, H, W, *x.stride(), xhi[GUARD:].data_ptr(),
                                         xlo[GUARD:].data_ptr(), amax[GUARD:].data_ptr(), st), 'c2m_conv3x3_operand_f32')
    xp = ops.PSA(xhi[GUARD:GUARD + npsa].view(B, c8i, H, W, 8), xlo[GUARD:GUARD + npsa].view(B, c8i, H, W, 8),
                 B, cin, H, W)
    y = _guarded(B * cout * H * W, torch.float32)
    a = _lib.ConvArgs()
    a.in_hi, a.in_lo, a.Cin, a.B, a.H, a.W = xp.hi.data_ptr(), xp.lo.data_ptr(), cin, B, H, W
    a.packed_w, a.bias, a.Cout = ops.conv3x3_pack_weights(w).data_ptr(), b.data_ptr(), cout
    a.out_f32, a.x_amax = y[GUARD:].data_ptr(), amax[GUARD:].data_ptr()
    a.os_b, a.os_c, a.os_y, a.os_x = cout * H * W, H * W, W, 1
    _lib.check(L.c2m_conv3x3(ctypes.addressof(a), st), 'c2m_conv3x3')
    gp, gamax = ops._conv3x3_operand(gy)
    nws = L.c2m_conv3x3_wgrad_workspace_bytes(B, cin, cout, H, W)
    ws, dw = _guarded(nws // 4, torch.float32), _guarded(cout * cin * 9, torch.float32)
    _lib.check(L.c2m_conv3x3_wgrad_scaled(gp.hi.data_ptr(), gp.lo.data_ptr(), gamax.data_ptr(), xp.hi.data_ptr(),
                                   xp.lo.data_ptr(), amax[GUARD:].data_ptr(), B, cin, cout, H, W,
                                   dw[GUARD:].data_ptr(), ws[GUARD:].data_ptr(), nws, st), 'c2m_conv3x3_wgrad_scaled')
    torch.cuda.synchronize()
    for buf, n in ((xhi, npsa), (xlo, npsa), (amax, B), (y, y_op.numel()), (ws, nws // 4), (dw, dw_op.numel())):
        assert _guards_intact(buf, n)
    assert torch.equal(y[GUARD:GUARD + y_op.numel()].view_as(y_op), y_op)
    assert torch.equal(dw[GUARD:GUARD + dw_op.numel()].view_as(dw_op), dw_op)
