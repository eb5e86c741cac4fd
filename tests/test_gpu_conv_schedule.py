"""Tensor-core 3x3 convolution at the edges of its CTA schedule (-m gpu).

Each CTA computes one 64-wide output-channel slice of every C-th 16x8-pixel tile of the batch, C being the number of
CTAs per slice, so tile counts per CTA differ by at most one.  On a 132-SM H100 a slice gets 132 / nslice CTAs (132,
66, 44, 33 for 1..4 slices), so the shapes below put the tile count below, at and just above that number, and leave
uneven remainders.  They cover weights that stay resident (Cin <= 64, one to four slices) and weights streamed per
tile (Cin > 64, two inputs), the specialised epilogue and the generic one (residual, PixelShuffle, octet fp32, partial
last slice), against fp64 at the bars of test_gpu_parity.py: 1e-5 (PSA output) and 3e-5 (general modes) of the
output scale.  The schedule must not change a single bit: a batch equals its images run one at a time."""
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


def _want(x1, x2, w, b, act):
    want = F.conv2d((torch.cat([x1, x2], 1) if x2 is not None else x1).double(), w.double(), b.double(), 1, 1)
    return want.relu() if act == 'relu' else F.leaky_relu(want, 0.1) if act == 'lrelu' else want


def _run(ops, p1, p2, wd, bd, act, mode, res):
    if mode == 'psa':
        return ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, residual=res))
    if mode == 'ps2':
        return ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, pixel_shuffle=2))
    if mode == 'oct':
        return ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, psa_out=False, out_f32=True, f32_octets=True).nchw()
    raise ValueError(mode)


# (B, Cin, Cin2, Cout, H, W, act, mode, residual)
CASES = [
    # one slice (132 CTAs): 4, 8, 132, 133 and 162 tiles; resident and streamed weights
    (1, 64, 0, 64, 18, 10, 'relu', 'psa', False),
    (2, 64, 0, 64, 19, 11, 'lrelu', 'psa', True),
    (3, 64, 0, 64, 64, 88, 'lrelu', 'psa', True),
    (1, 64, 0, 64, 112, 152, None, 'psa', False),
    (2, 32, 0, 64, 130, 70, 'relu', 'psa', False),
    (3, 3, 0, 48, 19, 11, 'lrelu', 'psa', False),
    (1, 96, 0, 64, 112, 152, 'relu', 'psa', True),
    (2, 64, 64, 64, 130, 70, 'lrelu', 'psa', False),
    # two slices (66 CTAs each): 65, 66, 68 tiles
    (1, 64, 0, 128, 80, 104, 'relu', 'psa', False),
    (1, 64, 0, 128, 96, 88, 'lrelu', 'psa', True),
    (1, 128, 0, 128, 64, 136, 'lrelu', 'psa', False),
    # three slices (44 CTAs each): 44, 45 tiles, partial last slice
    (1, 64, 0, 192, 64, 88, 'lrelu', 'psa', False),
    (1, 128, 0, 160, 80, 72, None, 'psa', False),
    # four slices (33 CTAs each): 8, 32, 33, 34 tiles
    (2, 64, 0, 256, 19, 11, 'lrelu', 'ps2', False),
    (1, 64, 0, 216, 64, 64, None, 'oct', False),
    (1, 64, 0, 256, 48, 88, 'lrelu', 'psa', True),
    (1, 64, 256, 256, 32, 136, 'lrelu', 'psa', False),
    (3, 64, 0, 216, 18, 10, None, 'oct', False),
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: f'B{c[0]}_{c[1]}+{c[2]}to{c[3]}_{c[4]}x{c[5]}_{c[7]}'
                                                      f'{"_res" if c[8] else ""}_t{_tiles(c[0], c[4], c[5])}')
def test_conv3x3_schedule_edges_vs_fp64(case):
    from c2m_b200 import ops
    B, c1, c2, cout, H, W, act, mode, res = case
    x1 = seeding.randn(21, (B, c1, H, W), 1.2)
    x2 = seeding.randn(22, (B, c2, H, W), 0.8) if c2 else None
    w = seeding.randn(23, (cout, c1 + c2, 3, 3), 0.03)
    b = seeding.randn(24, (cout,), 0.5)
    r = seeding.randn(25, (B, cout, H, W)) if res else None
    want = _want(x1, x2, w, b, act)
    if res:
        want = want + r.double()
    if mode == 'ps2':
        want = F.pixel_shuffle(want, 2)
    p1 = ops.psa_from_f32(x1.to(DEV))
    p2 = ops.psa_from_f32(x2.to(DEV)) if c2 else None
    rp = ops.psa_from_f32(r.to(DEV)) if res else None
    got = _run(ops, p1, p2, w.to(DEV), b.to(DEV), act, mode, rp)
    err = float((got.cpu().double() - want).abs().max())
    tol = 1e-5 if (mode == 'psa' and not c2 and c1 <= 64) else 3e-5
    assert err <= tol * float(want.abs().max()), err


@pytest.mark.parametrize('case', [(64, 0, 64, 64, 88, 'lrelu', 'psa', True), (128, 0, 128, 40, 56, 'relu', 'psa', False),
                                  (64, 0, 216, 48, 40, None, 'oct', False), (64, 0, 256, 19, 11, 'lrelu', 'ps2', False),
                                  (64, 64, 64, 130, 70, 'lrelu', 'psa', True)],
                         ids=lambda c: f'{c[0]}+{c[1]}to{c[2]}_{c[3]}x{c[4]}_{c[6]}{"_res" if c[7] else ""}')
def test_conv3x3_schedule_invariance_bitwise(case):
    """Which CTA computes a tile, and how many tiles it computes, must not change the result: a batch of 3 equals its
    images run one at a time (other tiles per CTA, other CTA counts), and two identical calls are equal."""
    from c2m_b200 import ops
    c1, c2, cout, H, W, act, mode, res = case
    B = 3
    x1 = ops.psa_from_f32(seeding.randn(31, (B, c1, H, W), 1.2).to(DEV))
    x2 = ops.psa_from_f32(seeding.randn(32, (B, c2, H, W), 0.8).to(DEV)) if c2 else None
    r = ops.psa_from_f32(seeding.randn(33, (B, cout, H, W)).to(DEV)) if res else None
    wd = seeding.randn(34, (cout, c1 + c2, 3, 3), 0.03).to(DEV)
    bd = seeding.randn(35, (cout,), 0.5).to(DEV)

    def one(i):
        def sl(p):
            return None if p is None else ops.PSA(p.hi[i:i + 1], p.lo[i:i + 1], 1, p.C, p.H, p.W, p.sa)
        return _run(ops, sl(x1), sl(x2), wd, bd, act, mode, sl(r))

    full = _run(ops, x1, x2, wd, bd, act, mode, r)
    again = _run(ops, x1, x2, wd, bd, act, mode, r)
    assert torch.equal(full, again)
    for i in range(B):
        assert torch.equal(full[i:i + 1], one(i)), i
