"""Pin the literal C restatement of `_ext.dcn_v2_forward` / `dcn_v2_backward` (oracle/c2m_oracle.c) against
torchvision's `deform_conv2d` with fp64 autograd at asymmetric geometry: kh != kw, sh != sw, ph != pw and dh != dw.

A swap of any of these pairs inside the oracle (the `k / kw` tap decomposition, the output-size formula, the per-axis
base position) would go unnoticed at square geometry, and every GPU test of the general-geometry DCN kernels
(tests/test_gpu_dcn_general.py) compares against this oracle.  Offsets are kept away from integer positions here
because the bilinear derivative is one-sided there and autograd picks the other side."""
import pytest
import torch

import seeding
from oracle import c_oracle, ref_path

# (kh, kw, sh, sw, ph, pw, dh, dw, B, C, dg, Cout, H, W)
CASES = [
    (1, 3, 1, 1, 0, 1, 1, 1, 2, 4, 1, 5, 7, 9),
    (3, 5, 2, 1, 1, 2, 1, 2, 1, 6, 2, 7, 11, 10),
    (5, 3, 1, 2, 2, 0, 3, 1, 1, 9, 3, 4, 14, 9),
    (3, 1, 1, 3, 0, 2, 2, 1, 2, 8, 4, 6, 10, 11),
    (2, 2, 1, 1, 0, 0, 1, 1, 1, 12, 4, 5, 8, 7),
    (3, 5, 2, 1, 1, 2, 1, 2, 1, 4, 4, 3, 9, 12),
    (5, 3, 1, 2, 2, 0, 3, 1, 2, 2, 1, 6, 13, 8),
]


def _case_id(c):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, dg, Cout, H, W = c
    return f'k{kh}x{kw}_s{sh}x{sw}_p{ph}x{pw}_d{dh}x{dw}_B{B}_C{C}dg{dg}_Co{Cout}_{H}x{W}'


def _out_hw(c):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, dg, Cout, H, W = c
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


@pytest.fixture(scope='module', autouse=True)
def _build_c_oracle():
    c_oracle.build()


@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_dcn_oracle_asymmetric_geometry_vs_torchvision_fp64(case):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, dg, Cout, H, W = case
    geo = (kh, kw, sh, sw, ph, pw, dh, dw)
    Ho, Wo = _out_hw(case)
    T = kh * kw
    seed = 17 * kh + 5 * kw + dg
    x = seeding.randn(seed, (B, C, H, W))
    wgt = seeding.randn(seed + 1, (Cout, C, kh, kw), 0.3)
    bias = seeding.randn(seed + 2, (Cout,))
    off = seeding.randn(seed + 3, (B, 2 * dg * T, Ho, Wo), 2.5)
    off = torch.where((off - off.round()).abs() < 0.05, off + 0.11, off)
    mask = torch.sigmoid(seeding.randn(seed + 4, (B, dg * T, Ho, Wo)))
    gout = seeding.randn(seed + 5, (B, Cout, Ho, Wo))

    leaves = [t.double().requires_grad_(True) for t in (x, wgt, bias, off, mask)]
    y = ref_path.dcn_v2_forward(leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], *geo, dg)
    assert tuple(y.shape) == (B, Cout, Ho, Wo)
    y.backward(gout.double())

    fwd = c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, *geo, dg=dg, acc64=True)
    want = y.detach()
    assert float((fwd.double() - want).abs().max()) <= 2e-5 * float(want.abs().max()), 'forward'

    gx, goff, gm, gw, gb = c_oracle.dcn_v2_backward(x, wgt, bias, off, mask, gout, *geo, dg)
    for got, leaf, name in ((gx, leaves[0], 'input'), (gw, leaves[1], 'weight'), (gb, leaves[2], 'bias'),
                            (goff, leaves[3], 'offset'), (gm, leaves[4], 'mask')):
        ref = leaf.grad
        assert float(ref.abs().max()) > 0, name
        assert float((got.double() - ref).abs().max()) <= 2e-5 * float(ref.abs().max()), name
