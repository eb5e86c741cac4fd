"""Deformable PS-ROI pooling on the CPU: the plain-C oracle (oracle/psroi_oracle.c) against an independent, vectorised
fp64 PyTorch restatement written here, known answers worked out by hand, the oracle's gradients against autograd of the
restatement, and the `_ext` / C ABI / module surface (names, rejected arguments, state-dict keys).

The restatement rounds ROI corners half away from zero (C `round`; `torch.round` rounds half to even), takes
`spatial_scale` and `trans_std` through float32 as the C signature does, and evaluates positions in the reference's
order, so in fp64 it takes the same skip / clamp branches as the oracle."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from oracle import psroi_oracle


def _rha(v):
    """C round(): half away from zero."""
    return torch.sign(v) * torch.floor(torch.abs(v) + 0.5)


def restate(x, bbox, trans, no_trans, scale, od, P, part, S, tstd, parts=False):
    """fp64 restatement -> (output, count) [R, od, P, P]; differentiable in x and trans.  With parts=True also returns
    the per-sample tensors the gradient checks need."""
    x, bbox = x.double(), bbox.double()
    scale, tstd = float(np.float32(scale)), float(np.float32(tstd))
    B, C, H, W = x.shape
    R = bbox.shape[0]
    K = 1 if no_trans else trans.shape[1] // 2
    cpc = od // K
    b = bbox[:, 0].to(torch.int64)                       # truncation toward zero
    bok = (b >= 0) & (b < B)
    sw = _rha(bbox[:, 1]) * scale - 0.5
    sh = _rha(bbox[:, 2]) * scale - 0.5
    rw = torch.clamp((_rha(bbox[:, 3]) + 1) * scale - 0.5 - sw, min=0.1)
    rh = torch.clamp((_rha(bbox[:, 4]) + 1) * scale - 0.5 - sh, min=0.1)
    bw, bh = rw / P, rh / P
    subw, subh = bw / S, bh / S
    p = torch.arange(P, dtype=torch.float64)
    pidx = torch.floor(p / P * part).long()
    cls = torch.arange(od) // cpc
    if no_trans:
        tx = ty = torch.zeros(R, od, P, P, dtype=torch.float64)
    else:
        t = trans.double()
        tx = t[:, 2 * cls][:, :, pidx[:, None], pidx[None, :]] * tstd
        ty = t[:, 2 * cls + 1][:, :, pidx[:, None], pidx[None, :]] * tstd
    v4 = lambda a: a[:, None, None, None]                 # noqa: E731
    ws = (p[None, None, None, :] * v4(bw) + v4(sw)) + tx * v4(rw)      # [R, od, ph, pw]
    hs = (p[None, None, :, None] * v4(bh) + v4(sh)) + ty * v4(rh)
    i = torch.arange(S, dtype=torch.float64)
    w = ws[..., None, None] + i[None, :] * v4(subw)[..., None, None]     # [..., ih, iw]
    h = hs[..., None, None] + i[:, None] * v4(subh)[..., None, None]
    w, h = torch.broadcast_tensors(w, h)
    keep = (w >= -0.5) & (w <= W - 0.5) & (h >= -0.5) & (h <= H - 0.5) & bok[:, None, None, None, None, None]
    wc, hc = w.clamp(0, W - 1), h.clamp(0, H - 1)
    x0, y0 = torch.floor(wc).detach().long(), torch.floor(hc).detach().long()
    x1, y1 = torch.ceil(wc).detach().long(), torch.ceil(hc).detach().long()
    lx, ly = wc - x0, hc - y0
    flat = x[b.clamp(0, max(B - 1, 0))].reshape(R, C, H * W)

    def g(yy, xx):
        return torch.gather(flat, 2, (yy * W + xx).reshape(R, od, -1)).view(yy.shape)
    v00, v01, v10, v11 = g(y0, x0), g(y1, x0), g(y0, x1), g(y1, x1)
    val = (1 - lx) * (1 - ly) * v00 + (1 - lx) * ly * v01 + lx * (1 - ly) * v10 + lx * ly * v11
    val = torch.where(keep, val, torch.zeros_like(val))
    cnt = keep.sum((-1, -2)).double()
    out = torch.where(cnt > 0, val.sum((-1, -2)) / cnt.clamp(min=1), torch.zeros_like(cnt))
    if parts:
        return out, cnt, dict(keep=keep, w=w, h=h, x0=x0, x1=x1, y0=y0, y1=y1, lx=lx, ly=ly, v=(v00, v01, v10, v11),
                              rw=rw, rh=rh, pidx=pidx, cls=cls, tstd=tstd, K=K)
    return out, cnt


def literal_trans_grad(gout, trans, cnt, pr, part):
    """The reference's trans-gradient rule, vectorised: it differentiates the bilinear blend at the CLAMPED position and
    ignores the clamp's own derivative."""
    R = gout.shape[0]
    diff = torch.where(cnt > 0, gout.double() / cnt.clamp(min=1), torch.zeros_like(cnt))[..., None, None]
    v00, v01, v10, v11 = [v.detach() for v in pr['v']]
    lx, ly = pr['lx'].detach(), pr['ly'].detach()
    k = pr['keep'].double()
    rw, rh = pr['rw'][:, None, None, None, None, None], pr['rh'][:, None, None, None, None, None]
    dx = (v11 * ly + v10 * (1 - ly) - v01 * ly - v00 * (1 - ly)) * pr['tstd'] * diff * rw * k
    dy = (v11 * lx + v01 * (1 - lx) - v10 * lx - v00 * (1 - lx)) * pr['tstd'] * diff * rh * k
    out = torch.zeros(R, 2 * pr['K'], part, part, dtype=torch.float64)
    od, P = gout.shape[1], gout.shape[2]
    for c in range(od):
        for ph in range(P):
            for pw in range(P):
                a, bb, cl = pr['pidx'][ph], pr['pidx'][pw], pr['cls'][c]
                out[:, 2 * cl, a, bb] += dx[:, c, ph, pw].sum((-1, -2))
                out[:, 2 * cl + 1, a, bb] += dy[:, c, ph, pw].sum((-1, -2))
    return out


def _args(no_trans, scale, od, P, part, S, tstd):
    return (int(no_trans), scale, od, 1, P, part, S, tstd)


def _case(seed, B, C, H, W, R, K, part, dtype=torch.float64, lo=-6.0, hi=None, dyadic=True):
    g = torch.Generator().manual_seed(seed)
    hi = max(H, W) + 6.0 if hi is None else hi
    x = torch.randn(B, C, H, W, generator=g, dtype=dtype)
    q = 4.0 if dyadic else 1.0
    corners = torch.floor((torch.rand(R, 4, generator=g, dtype=torch.float64) * (hi - lo) + lo) * q) / q
    bidx = torch.randint(0, B, (R, 1), generator=g).double()
    bbox = torch.cat([bidx, corners], 1).to(dtype)
    trans = (torch.floor(torch.randn(R, 2 * K, part, part, generator=g, dtype=torch.float64) * 64) / 64).to(dtype)
    return x, bbox, trans


# ---------------------------------------------------------------------------------------------- oracle vs restatement
@pytest.mark.parametrize('no_trans', [0, 1])
@pytest.mark.parametrize('P,part,S,K,scale,tstd', [(1, 1, 1, 1, 1.0, 0.1), (3, 3, 2, 3, 0.5, 0.1), (7, 7, 4, 1, 0.25, 0.1),
                                                   (3, 5, 7, 1, 1 / 3, 0.0), (7, 4, 2, 3, 1 / 16, 0.1)])
def test_oracle_matches_restatement_fp64(no_trans, P, part, S, K, scale, tstd):
    C = 6 * K
    x, bbox, trans = _case(P * 100 + S, 2, C, 9, 11, 7, K, part, hi=60.0 if scale < 0.1 else None,
                           dyadic=scale not in (1 / 3,))
    want_o, want_c = restate(x, bbox, trans, no_trans, scale, C, P, part, S, tstd)
    got_o, got_c = psroi_oracle.forward(x, bbox, trans, *_args(no_trans, scale, C, P, part, S, tstd))
    assert torch.equal(got_c, want_c)
    assert (got_c > 0).any() and (got_c == 0).any() or P == 1
    assert (got_o - want_o).abs().max() <= 1e-12 * max(1.0, want_o.abs().max())


def test_oracle_fp32_matches_restatement_on_dyadic_inputs():
    """Dyadic ROIs, scale and trans: every position is exact in fp32, so the fp32 instantiation counts the same."""
    x, bbox, trans = _case(5, 2, 6, 9, 11, 9, 2, 3)
    args = _args(0, 0.5, 6, 3, 3, 4, 0.25)
    want_o, want_c = restate(x, bbox, trans, *args[:2], 6, 3, 3, 4, 0.25)
    got_o, got_c = psroi_oracle.forward(x.float(), bbox.float(), trans.float(), *args)
    assert got_o.dtype == torch.float32 and torch.equal(got_c.double(), want_c)
    assert (got_o.double() - want_o).abs().max() <= 1e-6 * want_o.abs().max()


# ---------------------------------------------------------------------------------------------- known answers
def _pool(x, rois, P=1, S=2, scale=1.0, dtype=torch.float64):
    bbox = torch.tensor(rois, dtype=dtype)
    o, c = psroi_oracle.forward(x.to(dtype), bbox, torch.empty(0, dtype=dtype), *_args(1, scale, x.shape[1], P, P, S, 0.0))
    ro, rc = restate(x, bbox, None, 1, scale, x.shape[1], P, P, S, 0.0)
    assert torch.equal(c.double(), rc) and (o.double() - ro).abs().max() <= 1e-12 * max(1.0, ro.abs().max())
    return o, c


def _ramp(H, W, a=3.0, b=-2.0, d=0.5):
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing='ij')
    return (a * xx + b * yy + d)[None, None]


def test_constant_map_pools_to_the_constant():
    x = torch.full((1, 2, 8, 10), 2.75, dtype=torch.float64)
    _, _, trans = _case(1, 1, 2, 8, 10, 6, 2, 3)
    bbox = torch.tensor([[0, -9, -9, 4, 4], [0, 2, 1, 7, 6], [0, 6, 5, 30, 30], [0, 40, 40, 50, 50],
                         [0, 5, 5, 2, 2], [0, 3.5, 3.5, 3.5, 3.5]], dtype=torch.float64)
    for dtype in (torch.float32, torch.float64):
        o, c = psroi_oracle.forward(x.to(dtype), bbox.to(dtype), trans.to(dtype), *_args(0, 1.0, 2, 3, 3, 4, 0.5))
        assert (c > 0).any() and (c == 0).any()
        assert torch.equal(o[c > 0], torch.full_like(o[c > 0], 2.75)) and torch.equal(o[c == 0], torch.zeros_like(o[c == 0]))


def test_linear_ramp_gives_mean_of_clamped_sample_coordinates():
    """Bilinear interpolation is exact on a linear map, so a bin pools to a*mean(w) + b*mean(h) + d over its kept,
    clamped samples.  ROI (1,1)-(4,4) at scale 1: start 0.5, size 4, samples 0.5, 2.5 on each axis.  ROI (0,0)-(3,3):
    start -0.5, samples -0.5 (kept, clamped to 0) and 1.5.  ROI (5,0)-(9,3) on a 8-wide map: start 4.5, size 5, samples
    4.5 and 7.0 (x), -0.5 -> 0 and 1.5 (y)."""
    x = _ramp(6, 8)
    o, c = _pool(x, [[0, 1, 1, 4, 4], [0, 0, 0, 3, 3], [0, 5, 0, 9, 3]])
    want = [3.0 * 1.5 - 2.0 * 1.5 + 0.5, 3.0 * 0.75 - 2.0 * 0.75 + 0.5, 3.0 * 5.75 - 2.0 * 0.75 + 0.5]
    assert c.flatten().tolist() == [4, 4, 4]
    assert torch.allclose(o.flatten(), torch.tensor(want, dtype=torch.float64), rtol=0, atol=1e-12)


def test_roi_entirely_outside_gives_zero_and_count_zero():
    o, c = _pool(_ramp(6, 8), [[0, 20, 20, 30, 30], [0, -30, -30, -20, -20], [0, 20, 0, 30, 5], [0, 0, -9, 5, -3]],
                 P=2, S=3)
    assert torch.equal(c, torch.zeros_like(c)) and torch.equal(o, torch.zeros_like(o))


def test_exact_counts_at_each_border():
    """8x8 map, scale 1, P=2, S=2.  Left: x -3..3 -> samples -3.5, -1.75 | 0, 1.75 (first bin dropped).  Right: x 5..10
    -> 4.5, 6 | 7.5 (kept: on W - 0.5), 9 (dropped).  The y extent 2..5 keeps all four of its samples."""
    x = torch.ones(1, 1, 8, 8, dtype=torch.float64)
    _, c = _pool(x, [[0, -3, 2, 3, 5], [0, 5, 2, 10, 5], [0, 2, -3, 5, 3], [0, 2, 5, 5, 10]], P=2, S=2)
    assert c[0, 0].tolist() == [[0, 4], [0, 4]]
    assert c[1, 0].tolist() == [[4, 2], [4, 2]]
    assert c[2, 0].tolist() == [[0, 0], [4, 4]]
    assert c[3, 0].tolist() == [[4, 4], [2, 2]]


def test_inverted_and_zero_size_rois_get_size_point_one():
    """x2 < x1: start 4.5, size max(-2, 0.1) = 0.1.  x1 == x2 at scale 1/16: size 1/16 < 0.1 -> 0.1.  P=1, S=2 samples
    at start and start + 0.05."""
    x = _ramp(8, 8, a=1.0, b=0.0, d=0.0)
    o, c = _pool(x, [[0, 5, 5, 2, 2]])
    assert c.item() == 4 and abs(o.item() - (4.5 + 0.025)) < 1e-12
    o, c = _pool(x * 1.0, [[0, 48, 48, 48, 48]], scale=1 / 16)
    assert c.item() == 4 and abs(o.item() - (48 / 16 - 0.5 + 0.025)) < 1e-12


def test_half_coordinates_round_away_from_zero():
    """x1 = 2.5 -> 3, x2 = 4.5 -> 5, y1 = -0.5 -> -1, y2 = 2.5 -> 3: start (2.5, -1.5), size (3, 5); w samples 2.5 and
    4.0, h samples -1.5 (dropped) and 1.0.  Half-to-even rounding would keep four samples (h at -0.5 and 1.0)."""
    x = _ramp(8, 8, a=1.0, b=10.0, d=0.0)
    o, c = _pool(x, [[0, 2.5, -0.5, 4.5, 2.5]], S=2)
    assert c.item() == 2 and abs(o.item() - (3.25 + 10 * 1.0)) < 1e-12


def test_batch_index_truncates_and_out_of_range_pools_to_zero():
    x = torch.randn(2, 3, 6, 6, dtype=torch.float64)
    o, c = _pool(x, [[1.9, 1, 1, 4, 4], [-0.9, 1, 1, 4, 4], [2.0, 1, 1, 4, 4], [-1.0, 1, 1, 4, 4]])
    o1, _ = _pool(x[1:], [[0, 1, 1, 4, 4]])
    o0, _ = _pool(x[:1], [[0, 1, 1, 4, 4]])
    assert torch.equal(o[0], o1[0]) and torch.equal(o[1], o0[0])       # 1.9 -> 1, -0.9 -> 0
    assert torch.equal(c[2:], torch.zeros_like(c[2:])) and torch.equal(o[2:], torch.zeros_like(o[2:]))
    gx, _ = psroi_oracle.backward(torch.ones_like(o), x, torch.tensor([[2.0, 1, 1, 4, 4]], dtype=torch.float64),
                                  torch.empty(0, dtype=torch.float64), torch.ones(1, 3, 1, 1, dtype=torch.float64),
                                  *_args(1, 1.0, 3, 1, 1, 2, 0.0))
    assert torch.equal(gx, torch.zeros_like(gx))


# ---------------------------------------------------------------------------------------------- gradients
def _interior_case(seed, K=2, part=3, P=3, S=2, tstd=0.1):
    """ROIs well inside a 24x24 map with small translations: no sample is dropped or clamped."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4 * K, 24, 24, generator=g, dtype=torch.float64)
    x1 = torch.randint(4, 9, (5, 2), generator=g).double()
    sz = torch.randint(3, 9, (5, 2), generator=g).double()
    bbox = torch.cat([torch.randint(0, 2, (5, 1), generator=g).double(), x1, x1 + sz], 1)
    trans = torch.randn(5, 2 * K, part, part, generator=g, dtype=torch.float64) * 0.5
    return x, bbox, trans, (0, 1.0, 4 * K, P, part, S, tstd)


@pytest.mark.parametrize('seed', [0, 1])
def test_oracle_gradients_match_autograd_without_clamps(seed):
    x, bbox, trans, (nt, scale, od, P, part, S, tstd) = _interior_case(seed)
    xr, tr = x.clone().requires_grad_(), trans.clone().requires_grad_()
    out, cnt, pr = restate(xr, bbox, tr, nt, scale, od, P, part, S, tstd, parts=True)
    assert pr['keep'].all() and (pr['w'] > 0).all() and (pr['w'] < 23).all() and (pr['h'] > 0).all()
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed + 7), dtype=torch.float64)
    (out * gout).sum().backward()
    _, ocnt = psroi_oracle.forward(x, bbox, trans, nt, scale, od, 1, P, part, S, tstd)
    gx, gt = psroi_oracle.backward(gout, x, bbox, trans, ocnt, nt, scale, od, 1, P, part, S, tstd)
    assert (gx - xr.grad).abs().max() <= 1e-12 * xr.grad.abs().max()
    # autograd differentiates the trans_std-scaled translation through the float32-rounded trans_std, as the oracle
    assert (gt - tr.grad).abs().max() <= 1e-12 * tr.grad.abs().max()


def test_clamped_trans_gradient_follows_the_literal_rule():
    """Samples in (-0.5, 0) or (W-1, W-0.5) are clamped.  The reference differentiates the blend at the clamped
    position and ignores the clamp; the clamped coordinate is an integer there (floor == ceil), so that rule gives the
    axis a zero derivative, the same as the clamp's own."""
    x = torch.randn(1, 2, 6, 7, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    bbox = torch.tensor([[0, 0, 0, 6, 5], [0, -1, 1, 3, 4], [0, 3, -1, 6, 5]], dtype=torch.float64)
    trans = torch.tensor(np.random.default_rng(4).standard_normal((3, 2, 2, 2)) * 0.25)
    args = (0, 1.0, 2, 2, 2, 3, 0.125)
    out, cnt, pr = restate(x, bbox, trans, *args[:2], 2, 2, 2, 3, 0.125, parts=True)
    clamped = pr['keep'] & ((pr['w'] < 0) | (pr['w'] > 6) | (pr['h'] < 0) | (pr['h'] > 5))
    assert clamped.any()
    assert torch.equal(pr['x0'][clamped & ((pr['w'] < 0) | (pr['w'] > 6))],
                       pr['x1'][clamped & ((pr['w'] < 0) | (pr['w'] > 6))])
    gout = torch.randn(out.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    want = literal_trans_grad(gout, trans, cnt, pr, 2)
    _, ocnt = psroi_oracle.forward(x, bbox, trans, args[0], 1.0, 2, 1, 2, 2, 3, 0.125)
    _, gt = psroi_oracle.backward(gout, x, bbox, trans, ocnt, args[0], 1.0, 2, 1, 2, 2, 3, 0.125)
    assert (gt - want).abs().max() <= 1e-12 * want.abs().max()
    tr = trans.clone().requires_grad_()
    o2, _ = restate(x, bbox, tr, *args[:2], 2, 2, 2, 3, 0.125)
    (o2 * gout).sum().backward()
    assert (tr.grad - want).abs().max() <= 1e-12 * want.abs().max()


# ---------------------------------------------------------------------------------------------- surface
def test_ext_psroi_signatures():
    import _ext
    assert list(inspect.signature(_ext.dcn_v2_psroi_pooling_forward).parameters) == [
        'input', 'bbox', 'trans', 'no_trans', 'spatial_scale', 'output_dim', 'group_size', 'pooled_size', 'part_size',
        'sample_per_part', 'trans_std']                                                           # dcn_v2.h:75-86
    assert list(inspect.signature(_ext.dcn_v2_psroi_pooling_backward).parameters) == [
        'out_grad', 'input', 'bbox', 'trans', 'top_count', 'no_trans', 'spatial_scale', 'output_dim', 'group_size',
        'pooled_size', 'part_size', 'sample_per_part', 'trans_std']                               # dcn_v2.h:110-123


def test_ext_psroi_cpu_tensors_raise():
    import _ext
    x, bbox, trans = torch.zeros(1, 4, 6, 6), torch.zeros(2, 5), torch.zeros(2, 2, 3, 3)
    with pytest.raises(RuntimeError, match=r'must be a CUDA tensor \(Not implemented on the CPU\)'):
        _ext.dcn_v2_psroi_pooling_forward(x, bbox, trans, 0, 1.0, 4, 1, 3, 3, 2, 0.1)
    with pytest.raises(RuntimeError, match=r'must be a CUDA tensor \(Not implemented on the CPU\)'):
        _ext.dcn_v2_psroi_pooling_backward(torch.zeros(2, 4, 3, 3), x, bbox, trans, torch.zeros(2, 4, 3, 3), 0, 1.0,
                                           4, 1, 3, 3, 2, 0.1)


def _abi_shape(**kw):
    from c2m_b200 import _lib
    d = dict(B=1, C=4, H=6, W=6, R=2, no_trans=0, num_classes=2, spatial_scale=1.0, trans_std=0.1, output_dim=4,
             group_size=1, pooled_size=3, part_size=3, sample_per_part=2)
    d.update(kw)
    return _lib.PsroiShape(**d)


@pytest.mark.parametrize('kw,msg', [
    (dict(C=3), 'input channels and output channels must equal'),
    (dict(group_size=2), 'group_size must be 1'),
    (dict(num_classes=3), 'must be a multiple of the number of trans classes'),
    (dict(num_classes=0), 'trans must have 2 \\* K channels'),
    (dict(pooled_size=0), 'must be >= 1'),
    (dict(part_size=0), 'must be >= 1'),
    (dict(sample_per_part=0), 'must be >= 1'),
    (dict(sample_per_part=46), 'sample_per_part above 45'),
])
def test_abi_rejects_bad_arguments_before_any_launch(kw, msg):
    """The library checks every argument before touching memory: null pointers with a bad shape report the shape."""
    import re

    import __graft_entry__ as g
    g.build()
    from c2m_b200 import _lib
    L = _lib.lib()
    s = _abi_shape(**kw)
    for fn in (L.c2m_psroi_pooling_forward_f32, L.c2m_psroi_pooling_forward_f64):
        assert fn(None, None, None, ctypes.byref(s), None, None, None) == 1
        assert re.search(msg, L.c2m_last_error().decode())
    for fn in (L.c2m_psroi_pooling_backward_f32, L.c2m_psroi_pooling_backward_f64):
        assert fn(None, None, None, None, None, ctypes.byref(s), None, None, None, 0, None) == 1
        assert re.search(msg, L.c2m_last_error().decode())
    assert L.c2m_psroi_pooling_forward_f32(None, None, None, ctypes.byref(_abi_shape()), None, None, None) == 1
    assert b'null pointer' in L.c2m_last_error()
    assert L.c2m_psroi_pooling_forward_f32(None, None, None, ctypes.byref(_abi_shape(R=0)), None, None, None) == 0
    assert L.c2m_psroi_pooling_workspace_bytes(ctypes.byref(_abi_shape()), 8) == 2 * 4 * 9 * 2 * 8
    assert L.c2m_psroi_pooling_workspace_bytes(ctypes.byref(_abi_shape(no_trans=1)), 8) == 0


def test_oracle_rejects_what_the_library_rejects():
    x, bbox, trans = _case(0, 1, 4, 6, 6, 2, 2, 3)
    for args in ((0, 1.0, 3, 1, 3, 3, 2, 0.1), (0, 1.0, 4, 2, 3, 3, 2, 0.1), (0, 1.0, 4, 1, 0, 3, 2, 0.1)):
        with pytest.raises(RuntimeError, match='rc=1'):
            psroi_oracle.forward(x, bbox, trans, *args)


def test_dcn_pooling_state_dict_matches_reference():
    """Keys and shapes of the reference's DCNPooling (dcn_v2.py:344-372); last fc layer zero-initialised."""
    from mmsr.models.archs.DCNv2.dcn_v2 import DCNPooling, DCNv2Pooling, dcn_v2_pooling  # noqa: F401
    m = DCNPooling(1 / 16, 7, 32, False, part_size=7, sample_per_part=4, trans_std=0.1, deform_fc_dim=64)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == {'offset_mask_fc.0.weight': (64, 7 * 7 * 32), 'offset_mask_fc.0.bias': (64,),
                      'offset_mask_fc.2.weight': (64, 64), 'offset_mask_fc.2.bias': (64,),
                      'offset_mask_fc.4.weight': (7 * 7 * 3, 64), 'offset_mask_fc.4.bias': (7 * 7 * 3,)}
    assert m.offset_mask_fc[4].weight.abs().sum() == 0 and m.offset_mask_fc[4].bias.abs().sum() == 0
    assert m.deform_fc_dim == 64 and m.part_size == 7 and m.group_size == 1
    assert DCNPooling(0.5, 3, 8, True).state_dict() == {}
    assert DCNv2Pooling(0.5, 3, 8, True).part_size == 3
    sig = inspect.signature(DCNPooling.__init__).parameters
    assert {k: v.default for k, v in sig.items() if v.default is not inspect._empty} == dict(
        group_size=1, part_size=None, sample_per_part=4, trans_std=0.0, deform_fc_dim=1024)
