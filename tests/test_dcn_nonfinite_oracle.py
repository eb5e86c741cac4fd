"""The C oracles propagate a NaN / Inf input exactly as torchvision's fp64 `deform_conv2d` does (CPU).

tests/test_gpu_dcn_range.py compares the finiteness pattern of every GPU forward with these oracles.  A sample reads
its four bilinear corners only when the point is inside the window (-1 < h < H, -1 < w < W) and the corner inside the
image; it then multiplies each corner by its weight, so an in-bounds corner of weight 0 still carries a NaN or Inf
(0 * NaN = NaN), while a corner that is not read carries nothing.  The oracles must agree on that, element by
element, for the placements and offsets the GPU tests use."""
import numpy as np
import pytest
import torch
from torchvision.ops import deform_conv2d

import seeding
from oracle import c_oracle
from oracle import deform_conv_oracle as dco

B, C, COUT, DG, H, W = 2, 16, 24, 2, 13, 11
CH = 5
VALUES = {'nan': float('nan'), 'pinf': float('inf'), 'ninf': float('-inf')}
PLACES = {'corner00': (0, 0), 'cornerHW': (H - 1, W - 1), 'top_mid': (0, W // 2), 'interior': (H // 2, W // 2 - 1)}
CASES = [(w, v, o) for w in PLACES for v in VALUES for o in ('zero', 'frac')] + \
    [('offsets', v, o) for v in VALUES for o in ('zero', 'frac')]


@pytest.fixture(scope='module', autouse=True)
def _oracles_built():
    c_oracle.build()
    dco.build()


def _inputs(where, value, offsets, seed=700):
    x = seeding.randn(seed, (B, C, H, W))
    wgt = seeding.randn(seed + 1, (COUT, C, 3, 3), 1.0 / np.sqrt(9 * C))
    bias = seeding.randn(seed + 2, (COUT,))
    off = seeding.randn(seed + 3, (B, 18 * DG, H, W), 2.0) if offsets == 'frac' else torch.zeros(B, 18 * DG, H, W)
    mask = torch.sigmoid(seeding.randn(seed + 4, (B, 9 * DG, H, W)))
    if where == 'offsets':
        v = VALUES[value]
        off[0, 3, 2, 4] = v
        off[0, 16, H - 1, W - 1] = v
        off[1, 18 + 9, 5, 0] = v
    else:
        x[0, CH, PLACES[where][0], PLACES[where][1]] = VALUES[value]
    return x, wgt, bias, off, mask


def _torchvision(x, wgt, bias, off, mask):
    return deform_conv2d(x.double(), off.double(), wgt.double(), bias.double(), padding=1, mask=mask.double())


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(c))
def test_oracles_nonfinite_pattern_vs_torchvision_fp64(case):
    """A non-finite offset puts its sample outside the window (NaN fails every comparison), so the sample is 0 and
    the whole output stays finite.  torchvision's CPU kernel casts floor(NaN) to an index there, so those cases are
    checked against that closed form instead."""
    x, wgt, bias, off, mask = _inputs(*case)
    if case[0] == 'offsets':
        want = torch.ones(B, COUT, H, W, dtype=torch.bool)
    else:
        want = torch.isfinite(_torchvision(x, wgt, bias, off, mask))
        assert bool((~want).any())
    outs = {
        'c_oracle_acc64': c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, dg=DG, acc64=True),
        'c_oracle_acc32': c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, dg=DG, acc64=False),
        'deform_conv_f32': dco.forward(x, wgt, bias, off, mask, 3, 3, 1, 1, 1, 1, 1, 1, 1, DG),
        'deform_conv_f64': dco.forward(x.double(), wgt.double(), bias.double(), off.double(), mask.double(),
                                       3, 3, 1, 1, 1, 1, 1, 1, 1, DG),
    }
    for name, out in outs.items():
        assert torch.equal(torch.isfinite(out), want), name
    # DCNv1 (modulation 1) against torchvision without a mask
    v1 = dco.forward(x.double(), wgt.double(), None, off.double(), None, 3, 3, 1, 1, 1, 1, 1, 1, 1, DG)
    tv1 = want if case[0] == 'offsets' else torch.isfinite(deform_conv2d(x.double(), off.double(), wgt.double(), None,
                                                                         padding=1))
    assert torch.equal(torch.isfinite(v1), tv1)


@pytest.mark.parametrize('value', list(VALUES))
def test_nonfinite_at_origin_marks_a_2x2_block(value):
    """Hand-worked: zero offsets, 3x3 / pad 1.  Output (ho, wo) tap (i, j) samples the integer point
    (ho - 1 + i, wo - 1 + j).  x[0, 0] is read only by the point (0, 0) itself, as its (low, low) corner: the points
    (-1, .) and (., -1) lie on the window's open edge and are not sampled, and no other point has (0, 0) as a corner.
    The point (0, 0) is tap (1 - ho, 1 - wo), which exists for ho, wo in {0, 1}: exactly the 2x2 block of output rows
    0-1 x columns 0-1, in every output channel of image 0."""
    x, wgt, bias, off, mask = _inputs('corner00', value, 'zero')
    want = torch.ones(B, COUT, H, W, dtype=torch.bool)
    want[0, :, :2, :2] = False
    for out in (c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, dg=DG, acc64=True),
                dco.forward(x.double(), wgt.double(), bias.double(), off.double(), mask.double(),
                            3, 3, 1, 1, 1, 1, 1, 1, 1, DG),
                _torchvision(x, wgt, bias, off, mask)):
        assert torch.equal(torch.isfinite(out), want)
