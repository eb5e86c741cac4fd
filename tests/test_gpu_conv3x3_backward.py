"""Backward of the tensor-core 3x3 convolution (ops.conv3x3), -m gpu.

dX runs on conv3x3_wgmma_kernel with the rotated weights, dW on conv3x3_wgrad_kernel, both from grad_output stored as PSA
at a power-of-two scale chosen on the device.  Checked against fp64 (torch.nn.grad.conv2d_input / conv2d_weight in
float64): the max abs error of every gradient is at most max(1e-5 max|ref|, 2 x the error of cuDNN fp32 with TF32 off on
the same case).  The activation's mask is the op's own forward output (y > 0): the forward has its own tests, and a
pre-activation within rounding of 0 that changes sign is not a backward error.  Also: exact 2^k scaling, bitwise
repeatability, sentinel guards around every buffer the new entry points write, non-finite propagation, and one
RestorationNet training step on both paths."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

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


def _wgrad_ctas(B, cin, cout, H, W):
    """(K ranges, tiles) of conv3x3_wgrad_kernel: one wave of 132 / (slices x chunks) CTAs per K range."""
    pairs = -(-cout // 64) * -(-cin // 32)
    tiles = B * -(-H // 16) * -(-W // 8)
    return min(max(1, 132 // pairs), tiles), tiles


# (B, Cin, Cout, H, W, act).  The stage-3 training shapes (batch 9, GT 160: 64-channel maps at 40, 80 and 160), the
# concatenating head / offset convolutions (64 + C) -> 64 and -> C, conv_offset_mask C -> 216, the tails and conv_first;
# then odd sizes, batches 1..9, and tile counts below, at and above one wave of K ranges (132 tiles for 64 -> 64).
CASES = [
    (9, 64, 64, 40, 40, 'relu'), (9, 64, 64, 80, 80, None), (9, 64, 64, 160, 160, 'relu'),
    (9, 320, 64, 40, 40, 'lrelu'), (9, 320, 256, 40, 40, 'lrelu'),
    (9, 192, 64, 80, 80, 'lrelu'), (9, 192, 128, 80, 80, 'lrelu'),
    (9, 128, 64, 160, 160, 'lrelu'), (9, 128, 64, 160, 160, None),
    (9, 256, 216, 40, 40, None), (9, 128, 216, 80, 80, None), (9, 64, 216, 160, 160, None),
    (9, 64, 256, 40, 40, None), (9, 64, 256, 80, 80, None), (9, 64, 32, 160, 160, None), (9, 32, 3, 160, 160, None),
    (9, 3, 64, 40, 40, 'lrelu'),
    (1, 64, 64, 19, 11, 'relu'), (2, 48, 40, 130, 70, 'lrelu'), (3, 3, 48, 19, 11, None), (5, 96, 80, 33, 27, 'relu'),
    (1, 64, 64, 176, 96, None), (1, 64, 64, 192, 88, 'lrelu'), (1, 64, 64, 208, 96, None),
    (7, 16, 24, 18, 10, 'relu'),
]


def _ids(c):
    k, t = _wgrad_ctas(c[0], c[1], c[2], c[3], c[4])
    return f'B{c[0]}_{c[1]}to{c[2]}_{c[3]}x{c[4]}_{c[5]}_t{t}_k{k}'


def _inputs(case, seed):
    B, cin, cout, H, W, act = case
    x = seeding.randn(seed, (B, cin, H, W), 1.0).to(DEV)
    w = seeding.randn(seed + 1, (cout, cin, 3, 3), 1.0 / math.sqrt(9 * cin)).to(DEV)
    b = seeding.randn(seed + 2, (cout,), 0.1).to(DEV)
    # loss-sized gradients (an L1 mean over a stage-3 batch gives ~2^-19 per element)
    gy = seeding.randn(seed + 3, (B, cout, H, W), 2.0 ** -19).to(DEV)
    return x, w, b, gy


def _tc_grads(x, w, b, act, gy):
    from c2m_b200 import ops
    xr, wr, br = (t.detach().clone().requires_grad_() for t in (x, w, b))
    y = ops.conv3x3(xr, wr, br, act)
    y.backward(gy)
    return y.detach(), xr.grad, wr.grad, br.grad


def _masked(y, gy, act):
    if act == 'relu':
        return torch.where(y > 0, gy, 0.)
    if act == 'lrelu':
        return torch.where(y > 0, gy, gy * 0.1)
    return gy


def _grads_of(x, w, g):
    """(dX, dW, db) of a plain 3x3 / pad 1 convolution for the masked gradient g, in g's dtype (cuDNN)."""
    dx = torch.nn.grad.conv2d_input(x.shape, w.to(g.dtype), g, 1, 1)
    dw = torch.nn.grad.conv2d_weight(x.to(g.dtype), w.shape, g, 1, 1)
    return dx, dw, g.sum((0, 2, 3))


@pytest.mark.parametrize('case', CASES, ids=_ids)
def test_conv3x3_backward_vs_fp64(case):
    act = case[5]
    x, w, b, gy = _inputs(case, 100)
    y, dx, dw, db = _tc_grads(x, w, b, act, gy)
    g = _masked(y, gy, act)
    want = _grads_of(x.double(), w.double(), g.double())
    cudnn = _grads_of(x, w, g)
    for name, got, ref, c32 in zip(('dX', 'dW', 'db'), (dx, dw, db), want, cudnn):
        err = float((got.double() - ref).abs().max())
        err32 = float((c32.double() - ref).abs().max())
        bar = max(1e-5 * float(ref.abs().max()), 2 * err32)
        print(f'{_ids(case)} {name}: err {err:.3e} cudnn-fp32 {err32:.3e} scale {float(ref.abs().max()):.3e} '
              f'ratio {err / bar:.3f}')
        assert err <= bar, (name, err, err32)


@pytest.mark.parametrize('case', [(2, 64, 64, 40, 40, 'lrelu'), (1, 3, 48, 19, 11, 'relu'), (3, 96, 80, 33, 27, None)],
                         ids=_ids)
def test_grad_output_scaling_is_exact(case):
    """grad_output * 2^k gives exactly 2^k times every gradient: the PSA scale is a power of two chosen on the device."""
    act = case[5]
    x, w, b, gy = _inputs(case, 200)
    _, dx0, dw0, db0 = _tc_grads(x, w, b, act, gy)
    for k in (-40, -20, 0, 20):
        _, dx, dw, db = _tc_grads(x, w, b, act, gy * 2.0 ** k)
        for got, base in ((dx, dx0), (dw, dw0), (db, db0)):
            assert torch.equal(got, base * 2.0 ** k), k


@pytest.mark.parametrize('case', [(9, 64, 64, 80, 80, 'relu'), (2, 320, 256, 40, 40, 'lrelu')], ids=_ids)
def test_backward_is_bitwise_repeatable(case):
    x, w, b, gy = _inputs(case, 300)
    first = _tc_grads(x, w, b, case[5], gy)
    again = _tc_grads(x, w, b, case[5], gy)
    for a, c in zip(first, again):
        assert torch.equal(a, c)


GUARD = 4096


def _guarded(n, dtype):
    buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=dtype, device=DEV)
    if dtype == torch.float16:
        buf.fill_(-12345.0)
    return buf


def _guards_intact(buf, dtype):
    edge = torch.cat([buf[:GUARD], buf[-GUARD:]])
    return bool(edge.isnan().all()) if dtype == torch.float32 else bool((edge == -12345.0).all())


@pytest.mark.parametrize('case', [(2, 40, 72, 19, 11, None), (1, 64, 64, 130, 70, None), (3, 3, 3, 18, 10, None)],
                         ids=_ids)
def test_backward_with_per_image_grad_exponents_writes_stay_in_bounds(case):
    """Every buffer the backward's entry points write (the PSA gradient and its per-image amax from
    c2m_conv3x3_operand_f32, dW from the forward's per-image operand through c2m_conv3x3_wgrad_scaled, the workspace,
    dX from c2m_conv3x3 with the gradient's exponents) sits between sentinel guards that must come back untouched; the
    results must equal the op's."""
    from c2m_b200 import _lib, ops
    B, cin, cout, H, W, _ = case
    x, w, b, gy = _inputs(case, 400)
    _, dx_op, dw_op, _ = _tc_grads(x, w, b, None, gy)
    L = _lib.lib()
    c8o, c8i = (cout + 7) // 8, (cin + 7) // 8
    npsa = B * c8o * H * W * 8
    ghi, glo = _guarded(npsa, torch.float16), _guarded(npsa, torch.float16)
    amax = _guarded(B, torch.float32)
    st = torch.cuda.current_stream().cuda_stream
    rc = L.c2m_conv3x3_operand_f32(gy.data_ptr(), B, cout, H, W, *gy.stride(), ghi[GUARD:].data_ptr(),
                                   glo[GUARD:].data_ptr(), amax[GUARD:].data_ptr(), st)
    _lib.check(rc, 'c2m_conv3x3_operand_f32')
    xp, x_amax = ops._conv3x3_operand(x)
    assert xp.hi.numel() == B * c8i * H * W * 8
    nws = L.c2m_conv3x3_wgrad_workspace_bytes(B, cin, cout, H, W)
    ws = _guarded(nws // 4, torch.float32)
    dw = _guarded(cout * cin * 9, torch.float32)
    rc = L.c2m_conv3x3_wgrad_scaled(ghi[GUARD:].data_ptr(), glo[GUARD:].data_ptr(), amax[GUARD:].data_ptr(),
                             xp.hi.data_ptr(), xp.lo.data_ptr(), x_amax.data_ptr(), B, cin, cout, H, W,
                             dw[GUARD:].data_ptr(),
                             ws[GUARD:].data_ptr(), nws, st)
    _lib.check(rc, 'c2m_conv3x3_wgrad_scaled')
    dxs = _guarded(x.numel(), torch.float32)
    a = _lib.ConvArgs()
    a.in_hi, a.in_lo, a.Cin, a.B, a.H, a.W = ghi[GUARD:].data_ptr(), glo[GUARD:].data_ptr(), cout, B, H, W
    a.packed_w, a.Cout = ops.conv3x3_pack_weights(w, dgrad=True).data_ptr(), cin
    a.out_f32, a.x_amax = dxs[GUARD:].data_ptr(), amax[GUARD:].data_ptr()
    a.os_b, a.os_c, a.os_y, a.os_x = cin * H * W, H * W, W, 1
    _lib.check(L.c2m_conv3x3(ctypes.addressof(a), st), 'c2m_conv3x3')
    torch.cuda.synchronize()
    for buf, dt in ((ghi, torch.float16), (glo, torch.float16), (dw, torch.float32), (ws, torch.float32),
                    (dxs, torch.float32)):
        assert _guards_intact(buf, dt)
    assert bool(amax[:GUARD].isnan().all()) and bool(amax[GUARD + B:].isnan().all())
    assert torch.equal(dw[GUARD:GUARD + dw_op.numel()].view_as(dw_op), dw_op)
    assert torch.equal(dxs[GUARD:GUARD + x.numel()].view_as(dx_op), dx_op)


@pytest.mark.parametrize('bad', ['nan', 'inf', '-inf'])
@pytest.mark.parametrize('where', [(0, 12), (20, 6), (9, 12), (20, 12)], ids=['corner', 'last_row', 'last_col',
                                                                             'last_corner'])
def test_non_finite_grad_output_reaches_every_dependent_gradient(bad, where):
    """NaN / +-Inf in grad_output at a corner, in the last row or column of a 21 x 13 map (neither a multiple of the
    16 x 8 tile), plus an interior pixel: the finiteness patterns of dX, dW and db equal the fp64 reference's."""
    import conv3x3_ref
    case = (2, 40, 24, 21, 13, None)
    x, w, b, gy = _inputs(case, 500)
    gy[1, 5, where[0], where[1]] = float(bad)
    gy[0, 17, 9, 6] = float(bad)
    _, dx, dw, db = _tc_grads(x, w, b, None, gy)
    want = conv3x3_ref.conv3x3_grads(x, w, gy)
    for name, got, ref in zip(('dX', 'dW', 'db'), (dx, dw, db), want):
        assert bool((~torch.isfinite(ref)).any()), name
        assert torch.equal(torch.isfinite(got), torch.isfinite(ref)), name


def test_restoration_net_training_step_matches_cudnn(monkeypatch):
    """RestorationNet(64, 16, 8), B = 2, LR 40x40, pre-offsets and Ref features from net_map under no_grad, L1 loss:
    the tensor-core path launches the 3x3 kernel during the backward (none with C2M_FAST_CONV=0), and the parameters'
    gradients match the cuDNN fp32 path's in relative L2: within 1e-4 for the layers after the last deformable
    convolution (head_large, body_large, tail_large), within 1e-3 for every parameter.  The gradient of a bilinear
    sample with respect to its offset jumps where the sample crosses a pixel boundary, so the rounding-level forward
    difference between the paths moves a few samples across one and changes the gradients of everything upstream of
    the offsets by more than the convolutions' own error."""
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

    def step(fast):
        monkeypatch.setenv('C2M_FAST_CONV', '1' if fast else '0')
        net_g.zero_grad(set_to_none=True)
        loss = F.l1_loss(net_g(x, pre, feats), hr)
        torch.cuda.synchronize()
        ops.profile_enable(True)
        ops.profile_collect('conv3x3')
        loss.backward()
        torch.cuda.synchronize()
        launches = ops.profile_collect('conv3x3')['launches']
        ops.profile_enable(False)
        return launches, {n: p.grad.detach().clone() for n, p in net_g.named_parameters()}

    n_fast, g_fast = step(True)
    n_ref, g_ref = step(False)
    assert n_fast > 0 and n_ref == 0, (n_fast, n_ref)
    dist = {n: float((g_fast[n].double() - gr.double()).norm() / gr.double().norm().clamp_min(1e-300))
            for n, gr in g_ref.items()}
    after = {n: d for n, d in dist.items() if n.split('.')[1] in ('head_large', 'body_large', 'tail_large')}
    worst, worst_after = max(dist.items(), key=lambda kv: kv[1]), max(after.items(), key=lambda kv: kv[1])
    print(f'worst relative L2 gradient distance {worst[1]:.3e} at {worst[0]}; after the last DCN {worst_after[1]:.3e} '
          f'at {worst_after[0]}')
    assert worst_after[1] <= 1e-4, worst_after
    assert worst[1] <= 1e-3, worst
