"""Tensor-core 3x3 convolution: every branch of its epilogue call (-m gpu).

The epilogue is called with a constant residual pointer in each branch, so that the residual octets prefetched before
the MMAs stay in registers: specialised full blocks with and without a residual (PSA, octet fp32), the generic
epilogue with a residual (partial last column block, a second residual) and without one (strided fp32 output,
channels-last, PixelShuffle(2)), for every N (Cout 16 / 32 / 48 / 64 and more slices), resident and streamed weights, partial tiles at the
right and bottom edges, and runs of one or more 16x8 tiles per CTA.  Checked against fp64 at the bars of
test_gpu_conv_schedule.py: 1e-5 (PSA output) and 3e-5 (general modes) of the output scale."""
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


def _tiles(B, H, W):
    return B * ((H + 15) // 16) * ((W + 7) // 8)


# (B, Cin, Cin2, Cout, H, W, act, mode)
# modes: psa, res (one residual), res2 (two residuals), ps2 (PixelShuffle(2)), oct (octet-planar fp32),
#        f32 / f32cl (strided fp32 + add_f32, contiguous / channels-last)
CASES = [
    # specialised full blocks with a residual, each activation; 4 to 162 tiles on one slice
    (1, 64, 0, 64, 18, 10, 'relu', 'res'),
    (1, 64, 0, 64, 112, 152, 'lrelu', 'res'),
    (2, 64, 0, 64, 117, 155, None, 'res'),
    (1, 16, 0, 64, 53, 147, 'relu', 'res'),
    # generic epilogue with a residual: two residuals, partial last column block (Cout 48, 16), partial last slice
    (3, 64, 0, 64, 84, 90, 'lrelu', 'res2'),
    (2, 64, 0, 48, 95, 171, 'lrelu', 'res'),
    (2, 3, 0, 16, 19, 11, 'lrelu', 'res'),
    (1, 64, 0, 160, 45, 83, 'relu', 'res'),
    (1, 32, 32, 32, 84, 90, None, 'res'),
    # without a residual: specialised PSA / octet fp32, generic strided fp32 + add_f32, channels-last, PixelShuffle
    (1, 32, 0, 32, 53, 147, 'relu', 'psa'),
    (1, 64, 0, 64, 53, 147, 'relu', 'oct'),
    (2, 64, 0, 64, 95, 171, 'lrelu', 'f32'),
    (1, 64, 0, 48, 117, 155, None, 'f32cl'),
    (1, 64, 0, 256, 19, 83, 'lrelu', 'ps2'),
    # streamed weights (Cin > 64, two inputs) with and without a residual
    (1, 96, 0, 64, 53, 147, 'lrelu', 'res'),
    (1, 128, 0, 256, 45, 83, 'relu', 'res'),
    (1, 128, 0, 48, 95, 171, None, 'f32'),
    (2, 64, 64, 64, 19, 83, 'relu', 'psa'),
]


def _inputs(seed, B, c1, c2, cout, H, W, mode):
    x1 = seeding.randn(seed, (B, c1, H, W), 1.2)
    x2 = seeding.randn(seed + 1, (B, c2, H, W), 0.8) if c2 else None
    w = seeding.randn(seed + 2, (cout, c1 + c2, 3, 3), 0.03)
    b = seeding.randn(seed + 3, (cout,), 0.5)
    nres = {'res': 1, 'res2': 2}.get(mode, 0)
    res = [seeding.randn(seed + 4 + i, (B, cout, H, W)) for i in range(nres)]
    add = seeding.randn(seed + 6, (B, cout, H, W)) if mode in ('f32', 'f32cl') else None
    return x1, x2, w, b, res, add


def _want(x1, x2, w, b, act, mode, res, add):
    want = F.conv2d((torch.cat([x1, x2], 1) if x2 is not None else x1).double(), w.double(), b.double(), 1, 1)
    want = want.relu() if act == 'relu' else F.leaky_relu(want, 0.1) if act == 'lrelu' else want
    for r in res:
        want = want + r.double()
    if add is not None:
        want = want + add.double()
    return F.pixel_shuffle(want, 2) if mode == 'ps2' else want


def _run(ops, p1, p2, wd, bd, act, mode, res, add):
    """res: PSA residuals; add: fp32 tensor on the device."""
    if mode in ('psa', 'res', 'res2'):
        r1 = res[0] if res else None
        r2 = res[1] if len(res) > 1 else None
        return ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, residual=r1, residual2=r2))
    if mode == 'ps2':
        return ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, pixel_shuffle=2))
    if mode == 'oct':
        return ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, psa_out=False, out_f32=True, f32_octets=True).nchw()
    if mode in ('f32', 'f32cl'):
        cl = mode == 'f32cl'
        if cl:
            add = add.contiguous(memory_format=torch.channels_last)
        got = ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, psa_out=False, out_f32=True, add_f32=add, channels_last=cl)
        assert got.is_contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
        return got
    raise ValueError(mode)


def _case_id(c):
    return f'B{c[0]}_{c[1]}+{c[2]}to{c[3]}_{c[4]}x{c[5]}_{c[6]}_{c[7]}_t{_tiles(c[0], c[4], c[5])}'


@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_conv3x3_epilogue_branches_vs_fp64(case):
    from c2m_b200 import ops
    B, c1, c2, cout, H, W, act, mode = case
    x1, x2, w, b, res, add = _inputs(41, B, c1, c2, cout, H, W, mode)
    want = _want(x1, x2, w, b, act, mode, res, add)
    p1 = ops.psa_from_f32(x1.to(DEV))
    p2 = ops.psa_from_f32(x2.to(DEV)) if c2 else None
    rp = [ops.psa_from_f32(r.to(DEV)) for r in res]
    got = _run(ops, p1, p2, w.to(DEV), b.to(DEV), act, mode, rp, add.to(DEV) if add is not None else None)
    assert got.shape == want.shape
    err = float((got.cpu().double() - want).abs().max())
    tol = 1e-5 if (mode in ('psa', 'res', 'res2') and not c2 and c1 <= 64) else 3e-5
    assert err <= tol * float(want.abs().max()), err


# batches of 3 through each epilogue branch
BITWISE = [
    (64, 0, 64, 84, 90, 'lrelu', 'res'),
    (64, 0, 48, 53, 147, 'relu', 'res'),
    (64, 0, 64, 53, 147, 'lrelu', 'res2'),
    (64, 0, 256, 19, 83, 'lrelu', 'ps2'),
    (64, 0, 216, 37, 51, None, 'oct'),
    (32, 32, 48, 53, 147, 'relu', 'f32'),
    (128, 0, 64, 53, 147, 'lrelu', 'res'),
]


@pytest.mark.parametrize('case', BITWISE, ids=lambda c: f'{c[0]}+{c[1]}to{c[2]}_{c[3]}x{c[4]}_{c[6]}'
                                                       f'_t{_tiles(3, c[3], c[4])}')
def test_conv3x3_epilogue_branches_invariance_bitwise(case):
    """Which CTA computes a tile must not change the result: a batch of 3 equals its images run one at a time (other
    runs per CTA), and two identical calls are equal."""
    from c2m_b200 import ops
    c1, c2, cout, H, W, act, mode = case
    B = 3
    x1, x2, w, b, res, add = _inputs(51, B, c1, c2, cout, H, W, mode)
    p1 = ops.psa_from_f32(x1.to(DEV))
    p2 = ops.psa_from_f32(x2.to(DEV)) if c2 else None
    rp = [ops.psa_from_f32(r.to(DEV)) for r in res]
    ad = add.to(DEV) if add is not None else None
    wd, bd = w.to(DEV), b.to(DEV)

    def one(i):
        def sl(p):
            return None if p is None else ops.PSA(p.hi[i:i + 1], p.lo[i:i + 1], 1, p.C, p.H, p.W, p.sa)
        return _run(ops, sl(p1), sl(p2), wd, bd, act, mode, [sl(r) for r in rp],
                    ad[i:i + 1] if ad is not None else None)

    full = _run(ops, p1, p2, wd, bd, act, mode, rp, ad)
    again = _run(ops, p1, p2, wd, bd, act, mode, rp, ad)
    assert torch.equal(full, again)
    for i in range(B):
        assert torch.equal(full[i:i + 1], one(i)), i
