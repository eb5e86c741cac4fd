"""The ordered input-gradient oracle (oracle/ordered_grad_oracle.c) on the CPU.

It restates the summation order of the deterministic `grad_input` kernels (include/c2m_sm100.h, "ordered input
gradients").  Here it is checked two ways:
- bit for bit against a pure-numpy sequential loop in the same order and dtype;
- within 1e-6 (fp32) / 1e-13 (fp64) of the largest magnitude of the double-accumulating `grad_input` of
  oracle/deform_conv_oracle.c and oracle/psroi_oracle.c."""
import math

import numpy as np
import pytest
import torch

from oracle import deform_conv_oracle as dco
from oracle import ordered_grad_oracle as ogo
from oracle import psroi_oracle

F32, F64 = torch.float32, torch.float64
NP = {F32: np.float32, F64: np.float64}
BAR = {F32: 1e-6, F64: 1e-13}


@pytest.fixture(scope='module', autouse=True)
def _built():
    ogo.build()
    dco.build()
    psroi_oracle.build()


def _out_hw(geo, H, W):
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def _dcn_inputs(seed, B, C, Cout, groups, dg, H, W, geo, modulated):
    """Offsets are multiples of 1/64 (exact in both dtypes); a fifth of the sampling points sit on the border targets
    -1, 0, n-1 and n, and some fall outside the window."""
    kh, kw = geo[:2]
    Ho, Wo = _out_hw(geo, H, W)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g, dtype=F64)
    wgt = torch.randn(Cout, C // groups, kh, kw, generator=g, dtype=F64)
    off = torch.floor(torch.randn(B, 2 * dg * kh * kw, Ho, Wo, generator=g, dtype=F64) * 2 * 64) / 64
    sel = torch.rand(off.shape, generator=g) < 0.2
    tgt = torch.tensor([-1.0, 0.0, H - 1.0, float(H)])[torch.randint(0, 4, off.shape, generator=g)]
    off = torch.where(sel, tgt, off)                        # absolute targets, made relative below
    kk = torch.arange(kh * kw)
    base_h = (torch.arange(Ho) * geo[2] - geo[4])[None, :, None] + ((kk // kw) * geo[6])[:, None, None]
    base_w = (torch.arange(Wo) * geo[3] - geo[5])[None, None, :] + ((kk % kw) * geo[7])[:, None, None]
    o = off.view(B, dg, kh * kw, 2, Ho, Wo)
    s = sel.view(B, dg, kh * kw, 2, Ho, Wo)
    o[:, :, :, 0] = torch.where(s[:, :, :, 0], o[:, :, :, 0] - base_h, o[:, :, :, 0])
    o[:, :, :, 1] = torch.where(s[:, :, :, 1], o[:, :, :, 1] - base_w, o[:, :, :, 1])
    mask = None
    if modulated:
        mask = torch.floor(torch.randn(B, dg * kh * kw, Ho, Wo, generator=g, dtype=F64) * 64) / 64
        mask[torch.rand(mask.shape, generator=g) < 0.15] = 0.0
    gout = torch.randn(B, Cout, Ho, Wo, generator=g, dtype=F64)
    return x, wgt, off, mask, gout


def _gcol(wgt, gout, groups, T):
    """gcol [B, C*T, P] = grouped W^T gout, in fp64."""
    Cout = wgt.shape[0]
    B = gout.shape[0]
    wg = wgt.reshape(groups, Cout // groups, -1)
    gg = gout.reshape(B, groups, Cout // groups, -1)
    return torch.matmul(wg.transpose(1, 2), gg).reshape(B, -1, gg.shape[-1])


def _np_col2im(gcol, offset, mask, x_shape, geo, dg, dt):
    """Sequential loop: per element, ascending tap, output pixel, corner; adds in the dtype."""
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    B, C, H, W = x_shape
    Ho, Wo = _out_hw(geo, H, W)
    T, P, cpg = kh * kw, Ho * Wo, C // dg
    g = gcol.numpy().reshape(B, C, T, P)
    off = offset.numpy().reshape(B, dg, T, 2, P)
    m = None if mask is None else mask.numpy().reshape(B, dg, T, P)
    gx = np.zeros((B, C, H * W), dtype=dt)
    one = dt(1)
    for b in range(B):
        for c in range(C):
            grp = c // cpg
            for k in range(T):
                i, j = divmod(k, kw)
                for p in range(P):
                    ho, wo = divmod(p, Wo)
                    h = dt(ho * sh - ph + i * dh) + off[b, grp, k, 0, p]
                    w = dt(wo * sw - pw + j * dw) + off[b, grp, k, 1, p]
                    if not (h > -1 and w > -1 and h < H and w < W):
                        continue
                    hl, wl = int(math.floor(h)), int(math.floor(w))
                    lh, lw = h - dt(hl), w - dt(wl)
                    hh, hw = one - lh, one - lw
                    tg = g[b, c, k, p] * (one if m is None else m[b, grp, k, p])
                    for ok, y, x_, a, bb in ((hl >= 0 and wl >= 0, hl, wl, hh, hw),
                                             (hl >= 0 and wl + 1 <= W - 1, hl, wl + 1, hh, lw),
                                             (hl + 1 <= H - 1 and wl >= 0, hl + 1, wl, lh, hw),
                                             (hl + 1 <= H - 1 and wl + 1 <= W - 1, hl + 1, wl + 1, lh, lw)):
                        if ok:
                            gx[b, c, y * W + x_] = gx[b, c, y * W + x_] + tg * a * bb
    return torch.from_numpy(gx.reshape(B, C, H, W))


# (geometry (kh, kw, sh, sw, ph, pw, dh, dw), B, C, Cout, groups, dg, H, W)
DCN_CASES = [
    ((3, 3, 1, 1, 1, 1, 1, 1), 2, 6, 6, 3, 2, 6, 5),
    ((3, 2, 2, 1, 1, 0, 1, 2), 1, 8, 4, 2, 4, 7, 6),
    ((2, 2, 1, 1, 0, 0, 1, 1), 2, 9, 6, 3, 3, 5, 5),
    ((1, 3, 1, 2, 0, 1, 1, 1), 1, 4, 4, 1, 1, 4, 7),
]


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('modulated', [False, True], ids=['v1', 'modulated'])
@pytest.mark.parametrize('case', range(len(DCN_CASES)))
def test_ordered_col2im_equals_numpy_loop_and_double_oracle(case, modulated, dtype):
    geo, B, C, Cout, groups, dg, H, W = DCN_CASES[case]
    x, wgt, off, mask, gout = _dcn_inputs(10 + case, B, C, Cout, groups, dg, H, W, geo, modulated)
    x, wgt, off, gout = [t.to(dtype) for t in (x, wgt, off, gout)]
    mask = None if mask is None else mask.to(dtype)
    gcol = _gcol(wgt.double(), gout.double(), groups, geo[0] * geo[1]).to(dtype)
    got = ogo.deform_col2im(gcol, off, mask, x.shape, *geo, dg)
    want = _np_col2im(gcol, off, mask, tuple(x.shape), geo, dg, NP[dtype])
    assert got.dtype == dtype
    assert torch.equal(got, want)
    ref = dco.backward(x, wgt, off, mask, gout, *geo, groups, dg)[0].double()
    scale = float(ref.abs().max())
    assert scale > 0
    assert float((got.double() - ref).abs().max()) <= BAR[dtype] * scale


def test_ordered_col2im_keeps_signed_zero_of_zero_weight_corners():
    """A point on an integer position has in-image corners of weight 0: they add -0 or +0, and an element that only
    receives such contributions of a negative gradient stays +0 (+0 + -0 = +0)."""
    geo = (1, 1, 1, 1, 0, 0, 1, 1)
    off = torch.zeros(1, 2, 2, 2, dtype=F32)
    gcol = -torch.ones(1, 1, 4, dtype=F32)
    got = ogo.deform_col2im(gcol, off, None, (1, 1, 2, 2), *geo, 1)
    assert torch.equal(got, -torch.ones(1, 1, 2, 2))
    assert not torch.signbit(ogo.deform_col2im(gcol * 0, off, None, (1, 1, 2, 2), *geo, 1)).any()


def _round_away(v):
    return math.copysign(math.floor(abs(v) + 0.5), v)


def _np_psroi(gout, x_shape, bbox, trans, cnt, no_trans, scale, output_dim, group_size, P, part, S, tstd, dt):
    """Sequential loop over (ROI, channel, bin, sample, corner) with the positions' float / double promotions of the
    reference; adds in the dtype."""
    B, C, H, W = x_shape
    R = bbox.shape[0]
    K = 1 if no_trans else trans.shape[1] // 2
    cpc = output_dim // K
    g, bb, cn = gout.numpy(), bbox.numpy(), cnt.numpy()
    tr = None if no_trans else trans.numpy()
    sc, ts = dt(np.float32(scale)), dt(np.float32(tstd))
    gx = np.zeros((B, C, H * W), dtype=dt)
    one = dt(1)
    for n in range(R):
        b = int(bb[n, 0])
        if not (0 <= b < B):
            continue
        sw_ = dt(float(dt(_round_away(float(bb[n, 1]))) * sc) - 0.5)
        sh_ = dt(float(dt(_round_away(float(bb[n, 2]))) * sc) - 0.5)
        ew = dt(float(dt(_round_away(float(bb[n, 3])) + 1.0) * sc) - 0.5)
        eh = dt(float(dt(_round_away(float(bb[n, 4])) + 1.0) * sc) - 0.5)
        rw, rh = dt(max(float(ew - sw_), 0.1)), dt(max(float(eh - sh_), 0.1))
        bw, bh = rw / dt(P), rh / dt(P)
        subw, subh = bw / dt(S), bh / dt(S)
        for c in range(output_dim):
            cls = c // cpc
            for ph in range(P):
                for pw in range(P):
                    count = cn[n, c, ph, pw]
                    if count <= 0:
                        continue
                    parth = int(math.floor(dt(ph) / dt(P) * dt(part)))
                    partw = int(math.floor(dt(pw) / dt(P) * dt(part)))
                    tx = dt(0) if no_trans else tr[n, 2 * cls, parth, partw] * ts
                    ty = dt(0) if no_trans else tr[n, 2 * cls + 1, parth, partw] * ts
                    ws = dt(pw) * bw + sw_
                    ws = ws + tx * rw
                    hs = dt(ph) * bh + sh_
                    hs = hs + ty * rh
                    diff = g[n, c, ph, pw] / count
                    for ih in range(S):
                        for iw in range(S):
                            w = ws + dt(iw) * subw
                            h = hs + dt(ih) * subh
                            if float(w) < -0.5 or float(w) > W - 0.5 or float(h) < -0.5 or float(h) > H - 0.5:
                                continue
                            w = dt(min(max(float(w), 0.0), W - 1.0))
                            h = dt(min(max(float(h), 0.0), H - 1.0))
                            x0, x1, y0, y1 = math.floor(w), math.ceil(w), math.floor(h), math.ceil(h)
                            lx, ly = w - dt(x0), h - dt(y0)
                            hx, hy = one - lx, one - ly
                            for ok, y, x_, a, wb in ((True, y0, x0, hx, hy), (y1 != y0, y1, x0, hx, ly),
                                                     (x1 != x0, y0, x1, lx, hy), (x1 != x0 and y1 != y0, y1, x1, lx, ly)):
                                if ok:
                                    gx[b, c, y * W + x_] = gx[b, c, y * W + x_] + a * wb * diff
    return torch.from_numpy(gx.reshape(B, C, H, W))


# (B, C, H, W, R, K, P, part, S, scale, trans_std)
PS_CASES = [
    (2, 6, 7, 9, 6, 3, 3, 2, 2, 0.5, 0.1),
    (2, 4, 6, 5, 5, 1, 2, 2, 3, 0.25, 0.1),
    (1, 6, 5, 6, 4, 2, 3, 3, 2, 1.0, 0.0),
]


def _ps_inputs(seed, B, C, H, W, R, K, part, scale, dtype):
    """Half-integer ROI corners (some inverted or off the map), dyadic trans, batch indices that include -1, B and
    B + 0.5, and zero counts."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g, dtype=F64)
    span = torch.tensor([W / scale, H / scale], dtype=F64)
    c = torch.floor((torch.rand(R, 4, generator=g, dtype=F64) * 1.4 - 0.2) * span.repeat(2) * 2) / 2
    c[::4, 2:] = c[::4, :2] - 2
    b = torch.randint(0, B, (R, 1), generator=g).double()
    b[1::3] = torch.tensor([-1.0, float(B), B + 0.5])[torch.arange(len(b[1::3])) % 3][:, None]
    trans = torch.floor(torch.randn(R, 2 * K, part, part, generator=g, dtype=F64) * 64) / 64
    return x.to(dtype), torch.cat([b, c], 1).to(dtype), trans.to(dtype)


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('no_trans', [0, 1])
@pytest.mark.parametrize('case', range(len(PS_CASES)))
def test_ordered_psroi_equals_numpy_loop_and_double_oracle(case, no_trans, dtype):
    B, C, H, W, R, K, P, part, S, scale, tstd = PS_CASES[case]
    x, bbox, trans = _ps_inputs(20 + case, B, C, H, W, R, K, part, scale, dtype)
    args = (no_trans, scale, C, 1, P, part, S, tstd)
    _, cnt = psroi_oracle.forward(x, bbox, trans, *args)
    cnt = cnt.clone()
    cnt.view(-1)[::7] = 0                                   # zero counts contribute nothing
    cnt.view(-1)[3::11] = -1.0
    gout = torch.randn(cnt.shape, generator=torch.Generator().manual_seed(5), dtype=F64).to(dtype)
    got = ogo.psroi_grad_input(gout, x.shape, bbox, trans, cnt, *args)
    want = _np_psroi(gout, tuple(x.shape), bbox, trans, cnt, *args, NP[dtype])
    assert got.dtype == dtype
    assert torch.equal(got, want)
    ref = psroi_oracle.backward(gout, x, bbox, trans, cnt, *args)[0].double()
    scale_ = float(ref.abs().max())
    assert scale_ > 0
    assert float((got.double() - ref).abs().max()) <= BAR[dtype] * scale_
