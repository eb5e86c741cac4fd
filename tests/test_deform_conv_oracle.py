"""Pin the literal C restatement of grouped deformable convolution (oracle/deform_conv_oracle.c), which every GPU test
of `deform_conv_cuda` compares against, on the CPU:

- against torchvision's `deform_conv2d` with fp64 autograd (it takes conv groups through the weight shape and an
  optional mask): v1 and modulated, groups 1 to 4, deformable groups that cut across conv groups (C = 6, groups = 3,
  dg = 2 puts channels 2 and 3 of conv group 1 into different deformable groups), and the asymmetric geometries of
  test_dcn_geometry_oracle.py, where a swapped axis would show.  Offsets are kept away from integer positions: the
  bilinear derivative is one-sided there and autograd may pick the other side.
- bit for bit against the `_ext` oracle (oracle_dcn_v2_*) at groups = 1 with a mask, in fp32.

Bars: the fp32 oracle within 2e-5 and the fp64 oracle within 1e-10 of each result's largest magnitude."""
import pytest
import torch
from torchvision.ops import deform_conv2d

import seeding
from oracle import c_oracle, deform_conv_oracle as dco

# (kh, kw, sh, sw, ph, pw, dh, dw, B, C, Cout, groups, dg)
CASES = [
    (3, 3, 1, 1, 1, 1, 1, 1, 2, 6, 6, 3, 2),
    (1, 3, 1, 1, 0, 1, 1, 1, 2, 4, 6, 2, 1),
    (3, 5, 2, 1, 1, 2, 1, 2, 1, 6, 9, 3, 2),
    (5, 3, 1, 2, 2, 0, 3, 1, 1, 8, 4, 4, 2),
    (3, 1, 1, 3, 0, 2, 2, 1, 2, 8, 8, 4, 4),
    (2, 2, 1, 1, 0, 0, 1, 1, 1, 12, 6, 2, 3),
    (3, 3, 1, 1, 1, 1, 1, 1, 1, 4, 5, 1, 2),
]
H, W = 11, 10


def _case_id(c):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, Cout, groups, dg = c
    return f'k{kh}x{kw}_s{sh}x{sw}_p{ph}x{pw}_d{dh}x{dw}_B{B}_C{C}_Co{Cout}_g{groups}_dg{dg}'


@pytest.fixture(scope='module', autouse=True)
def _build_oracles():
    c_oracle.build()
    dco.build()


def _inputs(case, seed, modulated):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, Cout, groups, dg = case
    Ho, Wo = dco.out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw)
    T = kh * kw
    x = seeding.randn(seed, (B, C, H, W))
    wgt = seeding.randn(seed + 1, (Cout, C // groups, kh, kw), 0.3)
    bias = seeding.randn(seed + 2, (Cout,))
    off = seeding.randn(seed + 3, (B, 2 * dg * T, Ho, Wo), 2.5)
    off = torch.where((off - off.round()).abs() < 0.05, off + 0.11, off)
    mask = torch.sigmoid(seeding.randn(seed + 4, (B, dg * T, Ho, Wo))) * 1.5 - 0.2 if modulated else None
    gout = seeding.randn(seed + 5, (B, Cout, Ho, Wo))
    return x, wgt, bias, off, mask, gout


def _close(got, want, bar, what):
    scale = float(want.abs().max())
    assert scale > 0, what
    err = float((got.double() - want).abs().max())
    assert err <= bar * scale, f'{what}: max abs err {err:.3e} vs scale {scale:.3e}'


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
@pytest.mark.parametrize('modulated', [False, True], ids=['v1', 'modulated'])
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_deform_conv_oracle_vs_torchvision_fp64(case, modulated, dtype):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, Cout, groups, dg = case
    geo = (kh, kw, sh, sw, ph, pw, dh, dw)
    x, wgt, bias, off, mask, gout = _inputs(case, 40 + 7 * CASES.index(case), modulated)
    with_bias = modulated            # v1 has no bias in the reference's DeformConv
    leaves = [t.double().requires_grad_(True) for t in (x, wgt, bias, off)]
    if modulated:
        leaves.append(mask.double().requires_grad_(True))
    y = deform_conv2d(leaves[0], leaves[3], leaves[1], leaves[2] if with_bias else None, stride=(sh, sw),
                      padding=(ph, pw), dilation=(dh, dw), mask=leaves[4] if modulated else None)
    y.backward(gout.double())
    bar = 2e-5 if dtype == torch.float32 else 1e-10
    cast = lambda t: None if t is None else t.to(dtype)
    fwd = dco.forward(cast(x), cast(wgt), cast(bias) if with_bias else None, cast(off), cast(mask), *geo, groups, dg)
    assert fwd.dtype == dtype and tuple(fwd.shape) == tuple(y.shape)
    _close(fwd, y.detach(), bar, 'forward')
    gx, goff, gm, gw, gb = dco.backward(cast(x), cast(wgt), cast(off), cast(mask), cast(gout), *geo, groups, dg)
    assert (gm is None) == (not modulated)
    pairs = [(gx, leaves[0], 'input'), (gw, leaves[1], 'weight'), (goff, leaves[3], 'offset')]
    if with_bias:
        pairs.append((gb, leaves[2], 'bias'))
    if modulated:
        pairs.append((gm, leaves[4], 'mask'))
    for got, leaf, name in pairs:
        assert got.dtype == dtype, name
        _close(got, leaf.grad, bar, name)


@pytest.mark.parametrize('case', [c for c in CASES if c[11] == 1] + [(3, 5, 2, 1, 1, 2, 1, 2, 2, 6, 7, 1, 3)],
                         ids=_case_id)
def test_deform_conv_oracle_f32_equals_ext_oracle_bitwise(case):
    kh, kw, sh, sw, ph, pw, dh, dw, B, C, Cout, groups, dg = case
    geo = (kh, kw, sh, sw, ph, pw, dh, dw)
    x, wgt, bias, off, mask, gout = _inputs(case, 90, True)
    want = c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, *geo, dg=dg, acc64=True)
    assert torch.equal(dco.forward(x, wgt, bias, off, mask, *geo, 1, dg), want)
    got = dco.backward(x, wgt, off, mask, gout, *geo, 1, dg)
    want = c_oracle.dcn_v2_backward(x, wgt, bias, off, mask, gout, *geo, dg)
    for g_, w_, name in zip(got, want, ('input', 'offset', 'mask', 'weight', 'bias')):
        assert torch.equal(g_, w_), name


def test_deform_conv_oracle_rejects_bad_groups():
    x = torch.zeros(1, 6, 5, 5)
    off = torch.zeros(1, 18, 3, 3)
    with pytest.raises(RuntimeError, match='rc=1'):
        dco.forward(x, torch.zeros(4, 2, 3, 3), None, off, None, 3, 3, 1, 1, 0, 0, 1, 1, 3, 1)   # Cout % groups
    with pytest.raises(RuntimeError, match='rc=1'):
        dco.forward(x, torch.zeros(6, 6, 3, 3), None, off, None, 3, 3, 1, 1, 0, 0, 1, 1, 1, 4)   # C % dg
