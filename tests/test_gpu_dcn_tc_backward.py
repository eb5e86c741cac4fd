"""Backward of the tensor-core deformable convolution (ops.dcn_v2_tc), -m gpu.

grad_offset / grad_mask / grad_input come from dcn_dgrad_kernel, the weight gradient from dcn_wgrad_kernel.  Checked
against the fp64 oracle (c_oracle.dcn_v2_backward): the max abs error of every gradient is at most
max(1e-5 max|ref|, 2 x the error of `_ext.dcn_v2_backward` on the same inputs).  Also: exact 2^k scaling, per-image
scales, non-finite propagation, bitwise forward / repeatability / batch independence, sentinel guards, and one
RestorationNet training step with C2M_DCN_TC at 1 and 0."""
import ctypes

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


def _offsets(kind, seed, B, dg, H, W):
    if kind == 'pyr':        # pyramid of a random index map (far, integer) + N(0, 0.5^2) residuals
        far = torch.randint(-157, 158, (B, 1, 2, H, W), generator=torch.Generator().manual_seed(seed)).float()
        res = seeding.randn(seed + 1, (B, dg * 9, 2, H, W), 0.5)
        return (far.expand(B, dg * 9, 2, H, W) + res).reshape(B, 18 * dg, H, W)
    if kind == 'small':
        return seeding.randn(seed, (B, 18 * dg, H, W), 2.0)
    # 'border': integer offsets that put sampling points on the first / last row and column
    g = torch.Generator().manual_seed(seed)
    ys = torch.arange(H).view(1, 1, H, 1).float()
    xs = torch.arange(W).view(1, 1, 1, W).float()
    ty = torch.randint(0, 2, (B, dg * 9, 1, 1), generator=g).float() * (H - 1)
    tx = torch.randint(0, 2, (B, dg * 9, 1, 1), generator=g).float() * (W - 1)
    k = torch.arange(9).view(1, 1, 9, 1, 1).repeat(1, dg, 1, 1, 1).view(1, dg * 9, 1, 1)
    oy = ty - ys - (k // 3 - 1).float()
    ox = tx - xs - (k % 3 - 1).float()
    return torch.stack((oy.expand(B, -1, H, W), ox.expand(B, -1, H, W)), 2).reshape(B, 18 * dg, H, W)


def _inputs(case, seed=0):
    B, C, cout, H, W, dg, ok, mk = case
    x = seeding.randn(seed, (B, C, H, W)).to(DEV)
    off = _offsets(ok, seed + 2, B, dg, H, W).to(DEV)
    mask = seeding.randn(seed + 3, (B, dg * 9, H, W))
    mask = (torch.sigmoid(mask) if mk == 'sig' else (mask * 3).clamp(-3, 3)).to(DEV)
    w = seeding.randn(seed + 4, (cout, C, 3, 3), (9 * C) ** -0.5).to(DEV)
    b = seeding.randn(seed + 5, (cout,), 0.1).to(DEV)
    gy = seeding.randn(seed + 6, (B, cout, H, W), 2.0 ** -19).to(DEV)
    return x, off, mask, w, b, gy


def _tc(x, off, mask, w, b, gy, x_grad=True):
    from c2m_b200 import ops
    xr = x.detach().clone().requires_grad_(x_grad)
    orr, mr, wr, br = (t.detach().clone().requires_grad_() for t in (off, mask, w, b))
    y = ops.dcn_v2_tc(xr, orr, mr, wr, br, off.shape[1] // 18)
    y.backward(gy)
    return y.detach(), (xr.grad if x_grad else None), orr.grad, mr.grad, wr.grad, br.grad


# (B, C, Cout, H, W, dg, offsets, mask): the stage-3 training shapes, odd maps and batches, C/dg = 8..64 (and a
# non-power-of-two 24), Cout partial and multiple slices, far / small / border offsets, masks in [-3, 3]
CASES = [
    (9, 256, 256, 40, 40, 8, 'pyr', 'sig'), (9, 128, 128, 80, 80, 8, 'pyr', 'sig'), (9, 64, 64, 160, 160, 8, 'pyr', 'sig'),
    (1, 64, 64, 19, 11, 8, 'small', 'sig'), (3, 64, 40, 33, 27, 4, 'small', 'pm3'), (2, 48, 72, 130, 70, 2, 'small', 'sig'),
    (5, 64, 16, 19, 11, 8, 'border', 'sig'), (7, 128, 200, 33, 27, 8, 'pyr', 'pm3'), (4, 96, 64, 24, 16, 4, 'small', 'sig'),
    (2, 128, 256, 24, 16, 2, 'border', 'pm3'), (6, 64, 72, 19, 11, 1, 'small', 'sig'),
    # column counts C * 9 that are not a multiple of dcn_dgrad_kernel's chunk width (a partial last chunk)
    (2, 32, 32, 19, 11, 1, 'small', 'sig'), (2, 32, 32, 19, 11, 4, 'pyr', 'pm3'), (3, 96, 64, 19, 11, 3, 'small', 'sig'),
    (2, 24, 16, 19, 11, 1, 'border', 'sig'),
]


def _ids(c):
    return f'B{c[0]}_{c[1]}to{c[2]}_{c[3]}x{c[4]}_dg{c[5]}_{c[6]}_{c[7]}'


def _err(a, ref):
    return float((a.double() - ref.double()).abs().max())


@pytest.mark.parametrize('case', CASES, ids=[_ids(c) for c in CASES])
def test_gradients_match_fp64_oracle(case):
    from c2m_b200 import ops
    from oracle import c_oracle
    x, off, mask, w, b, gy = _inputs(case)
    dg = case[5]
    ref = c_oracle.dcn_v2_backward(x.cpu().double(), w.cpu().double(), b.cpu().double(), off.cpu().double(),
                                   mask.cpu().double(), gy.cpu().double(), dg=dg)
    ext = ops.dcn_v2_backward(x, w, b, off, mask, gy, 3, 3, 1, 1, 1, 1, 1, 1, dg)
    names = ('grad_input', 'grad_offset', 'grad_mask', 'grad_weight', 'grad_bias')
    worst = 0.0
    for x_grad in (True, False):
        _, *mine = _tc(x, off, mask, w, b, gy, x_grad)
        for i, n in enumerate(names):
            if mine[i] is None:
                continue
            r = ref[i].to(DEV)
            bar = max(1e-5 * float(r.abs().max()), 2 * _err(ext[i], r))
            e = _err(mine[i], r)
            worst = max(worst, e / bar if bar > 0 else 0.0)
            assert e <= bar, (n, x_grad, e, bar)
    print(f'{_ids(case)}: worst error / bar {worst:.3f}')


def test_forward_bitwise_and_scaling():
    from c2m_b200 import ops
    case = (3, 64, 64, 33, 27, 8, 'small', 'sig')
    x, off, mask, w, b, gy = _inputs(case, 7)
    y, gx, go, gm, gw, gb = _tc(x, off, mask, w, b, gy)
    assert torch.equal(y, ops.dcn_v2_forward(x, w, b, off, mask, 3, 3, 1, 1, 1, 1, 1, 1, 8))
    # repeatability of everything but the atomically summed grad_input
    r = _tc(x, off, mask, w, b, gy)
    for a, c in zip((go, gm, gw, gb), r[2:]):
        assert torch.equal(a, c)
    # grad_output * 2^k: every gradient but grad_input exactly 2^k times
    r = _tc(x, off, mask, w, b, gy * 2.0 ** 37)
    for a, c in zip((go, gm, gw, gb), r[2:]):
        assert torch.equal(a * 2.0 ** 37, c)
    # x * 2^k: dW, grad_offset and grad_mask exactly 2^k times
    r = _tc(x * 2.0 ** -45, off, mask, w, b, gy)
    assert torch.equal(gw * 2.0 ** -45, r[4]) and torch.equal(go * 2.0 ** -45, r[2]) and torch.equal(gm * 2.0 ** -45, r[3])
    # batch independence of grad_offset / grad_mask
    for i in range(3):
        s = _tc(x[i:i + 1], off[i:i + 1], mask[i:i + 1], w, b, gy[i:i + 1])
        assert torch.equal(s[2], go[i:i + 1]) and torch.equal(s[3], gm[i:i + 1])


@pytest.mark.parametrize('amax', [(1e-30,), (1e30,), (1.0, 1e-5, 1e5)], ids=['tiny', 'huge', 'mixed'])
def test_range_each_image_to_its_own_scale(amax):
    """x at the ends of fp32's range and a batch of mixed magnitudes, held to the accuracy bar of
    test_gradients_match_fp64_oracle image by image for the per-image gradients (grad_input, grad_offset, grad_mask),
    over the batch for dW and db."""
    from c2m_b200 import ops
    from oracle import c_oracle
    case = (len(amax), 64, 64, 24, 16, 8, 'small', 'sig')
    x, off, mask, w, b, gy = _inputs(case, 11)
    x = x * torch.tensor(amax, device=DEV).view(-1, 1, 1, 1)
    _, *mine = _tc(x, off, mask, w, b, gy)
    ref = c_oracle.dcn_v2_backward(x.cpu().double(), w.cpu().double(), b.cpu().double(), off.cpu().double(),
                                   mask.cpu().double(), gy.cpu().double(), dg=8)
    ext = ops.dcn_v2_backward(x, w, b, off, mask, gy, 3, 3, 1, 1, 1, 1, 1, 1, 8)

    def check(got, e, r, what):
        r = r.to(DEV)
        bar = max(1e-5 * float(r.abs().max()), 2 * _err(e, r))
        assert _err(got, r) <= bar, (what, _err(got, r), bar)
    for i, a in enumerate(amax):
        for k, n in ((0, 'grad_input'), (1, 'grad_offset'), (2, 'grad_mask')):
            check(mine[k][i], ext[k][i], ref[k][i], (n, i, a))
    check(mine[3], ext[3], ref[3], 'grad_weight')
    check(mine[4], ext[4], ref[4], 'grad_bias')


@pytest.mark.parametrize('where', ['x', 'offset', 'grad_output'])
def test_nonfinite_pattern_matches_oracle(where):
    from oracle import c_oracle
    case = (2, 64, 64, 19, 11, 8, 'small', 'sig')
    x, off, mask, w, b, gy = _inputs(case, 21)
    t = {'x': x, 'offset': off, 'grad_output': gy}[where]
    t.view(-1)[5] = float('nan')
    t.view(-1)[t.numel() // 2 + 3] = float('inf')
    H, W = case[3], case[4]
    t[0, 7, H - 1, W - 1] = float('-inf')          # the last row and column of the map
    t[1, 2, H - 1, W // 2] = float('nan')
    _, *mine = _tc(x, off, mask, w, b, gy)
    ref = c_oracle.dcn_v2_backward(x.cpu().double(), w.cpu().double(), b.cpu().double(), off.cpu().double(),
                                   mask.cpu().double(), gy.cpu().double(), dg=8)
    for m, r in zip(mine, ref):
        assert torch.equal(torch.isfinite(m).cpu(), torch.isfinite(r)), where


def test_no_writes_outside_buffers_per_image_grad():
    """Sentinels around grad_output's per-image amax, and around grad_offset, grad_mask, grad_input and grad_weight of
    both entry points."""
    from c2m_b200 import _lib, ops
    L = _lib.lib()
    case = (2, 64, 40, 19, 11, 8, 'small', 'sig')
    x, off, mask, w, b, gy = _inputs(case, 31)
    B, C, H, W, cout, dg = 2, 64, 19, 11, 40, 8
    pad = 4096
    gp = ops.PSA.empty(B, cout, H, W, DEV)
    gamax_full = torch.full((B + 2 * pad,), -12345, dtype=torch.int32, device=DEV)
    gamax = gamax_full[pad:pad + B]
    _lib.check(L.c2m_conv3x3_operand_f32(gy.data_ptr(), B, cout, H, W, *gy.stride(), gp.hi.data_ptr(),
                                         gp.lo.data_ptr(), gamax.data_ptr(), ops._stream()), 'psa')
    x_il = torch.empty(L.c2m_dcn_tc_operand_bytes(B, C, H, W, dg) // 2, dtype=torch.float16, device=DEV)
    amax = torch.empty(2 * B, dtype=torch.int32, device=DEV)
    _lib.check(L.c2m_dcn_tc_operand_f32(x.data_ptr(), B, C, H, W, *x.stride(), dg, mask.data_ptr(), x_il.data_ptr(),
                                        amax.data_ptr(), ops._stream()), 'operand')

    def guarded(n):
        t = torch.full((n + 2 * pad,), 12345.0, device=DEV)
        return t, t[pad:pad + n]
    bufs = {k: guarded(n) for k, n in (('goff', off.numel()), ('gm', mask.numel()), ('gx', x.numel()),
                                       ('gw', w.numel()))}
    bufs['gx'][1].zero_()
    a = _lib.DcnTcGradArgs()
    a.gy_hi, a.gy_lo, a.gy_amax = gp.hi.data_ptr(), gp.lo.data_ptr(), gamax.data_ptr()
    a.x_il, a.x_amax, a.mask_amax = x_il.data_ptr(), amax.data_ptr(), amax.data_ptr() + 4 * B
    a.offset, a.mask = off.data_ptr(), mask.data_ptr()
    a.B, a.C, a.H, a.W, a.Cout, a.dg = B, C, H, W, cout, dg
    a.packed_w = ops._dcn_tc_pack_dgrad(w, dg).data_ptr()
    a.grad_offset, a.grad_mask, a.grad_input = (bufs[k][1].data_ptr() for k in ('goff', 'gm', 'gx'))
    _lib.check(L.c2m_dcn_tc_dgrad(ctypes.addressof(a), ops._stream()), 'dgrad')
    n = L.c2m_dcn_tc_wgrad_workspace_bytes(B, C, H, W, cout, dg)
    ws_full = torch.full((n // 4 + 2 * pad,), 12345.0, device=DEV)
    a.grad_weight, a.ws, a.ws_bytes = bufs['gw'][1].data_ptr(), ws_full[pad:].data_ptr(), n
    _lib.check(L.c2m_dcn_tc_wgrad(ctypes.addressof(a), ops._stream()), 'wgrad')
    torch.cuda.synchronize()
    for k, (full, _) in bufs.items():
        assert bool((full[:pad] == 12345.0).all()) and bool((full[-pad:] == 12345.0).all()), k
    assert bool((ws_full[:pad] == 12345.0).all()) and bool((ws_full[pad + n // 4:] == 12345.0).all())
    assert bool((gamax_full[:pad] == -12345).all()) and bool((gamax_full[pad + B:] == -12345).all())


def _training_setup():
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
    return net_g, x, hr, pre, feats


def _step(net_g, x, hr, pre, feats, monkeypatch, tc):
    from c2m_b200 import _lib, ops
    monkeypatch.setenv('C2M_DCN_TC', '1' if tc else '0')
    L = _lib.lib()
    calls = []
    for name in ('c2m_deform_conv_col2im_coord_f32', 'c2m_deform_conv_im2col_f32', 'c2m_deform_conv_col2im_f32',
                 'c2m_deform_conv_col2im_det_f32'):
        fn = getattr(L, name)
        monkeypatch.setattr(L, name, lambda *a, _fn=fn, _n=name: calls.append(_n) or _fn(*a), raising=False)
    net_g.zero_grad(set_to_none=True)
    loss = F.l1_loss(net_g(x, pre, feats), hr)
    torch.cuda.synchronize()
    ops.profile_enable(True)
    ops.profile_collect('dcn_dgrad')
    ops.profile_collect('dcn_wgrad')
    loss.backward()
    torch.cuda.synchronize()
    n_new = ops.profile_collect('dcn_dgrad')['launches'] + ops.profile_collect('dcn_wgrad')['launches']
    ops.profile_enable(False)
    monkeypatch.undo()
    return loss.detach(), n_new, calls, {n: p.grad.detach().clone() for n, p in net_g.named_parameters()}


def test_restoration_net_training_step(monkeypatch):
    """RestorationNet(64, 16, 8), B = 2, LR 40x40, set up as the 3x3 convolution's training-step test: the loss is
    bit-identical with C2M_DCN_TC at 1 and 0, the new kernels run only at 1 and the `_ext` backward pieces only at 0,
    and every parameter gradient agrees within 1e-4 relative L2."""
    args = _training_setup()
    l1, n1, c1, g1 = _step(*args, monkeypatch, True)
    l0, n0, c0, g0 = _step(*args, monkeypatch, False)
    assert torch.equal(l1, l0)
    assert n1 == 6 and not c1, (n1, c1)           # three DCNs x (dgrad, wgrad)
    assert n0 == 0 and c0, (n0, c0)
    dist = {n: float((g1[n].double() - g.double()).norm() / g.double().norm().clamp_min(1e-300)) for n, g in g0.items()}
    worst = max(dist.items(), key=lambda kv: kv[1])
    print(f'worst relative L2 gradient distance {worst[1]:.3e} at {worst[0]}')
    assert worst[1] <= 1e-4, worst


def test_training_step_deterministic(monkeypatch):
    args = _training_setup()
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        _, n1, c1, g1 = _step(*args, monkeypatch, True)
        _, n2, c2, g2 = _step(*args, monkeypatch, True)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    assert n1 == 6 and n2 == 6 and not c1 and not c2
    dcn = [n for n in g1 if '_dyn_agg.' in n]
    assert dcn
    for n in dcn:
        assert torch.equal(g1[n], g2[n]), n
