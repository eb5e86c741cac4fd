"""Tensor-core DCN (`dcn_wgmma_kernel`, csrc/dcn_umma.cu) at the configurations the model does not send (-m gpu).

The kernel's K axis is (group g, tap, channel octet): opp = C/dg/8 octets per (g, tap) pair, 4 octets per pipeline
stage, nkc = ceil(9 C/8 / 4) stages.  A gather thread fills L consecutive octets of one stage: L = opp (capped at 4)
when opp is a power of two (the pair is `ko >> opp_shift`), else L = 1 and the pair is `ko / opp`.  Ring depth 4
(L = 1) or 8 (L = 2, 4).  The MMA width N is Cout rounded up to 16 when Cout <= 64, else 64 per output slice.  The
pre-offsets come from a `pre_offset` tensor, from an index map through a per-tile flow table (scale 1, 2, 4, 8) or
from an index map decoded in place (any other scale; `fast_div` by the scale and by `ref_gw`).

Each case of CASES is compared with the fp64-accumulating C oracle at 2e-5 of the output scale.  Its id names what it
pins: C/dg, opp, L, nkc, N and slice count, offset source, om layout, outputs, map size and tile count.
- `C8_opp1_L1_nkc3_N16x1_om-only_nobias_5x3`: a map smaller than one 16x8 tile, no pre-offsets, bias None.
- `C24_opp3_L1_nkc7_N32x1_idx-s1-table`: opp not a power of two (`/ opp`), the N = 32 instantiation, scale-1 table.
- `C48dg2_opp3_L1_nkc14_N48x1_idx-s3-decode_psa`: in-place decode (scale 3), PSA and fp32 outputs.
- `C64_opp8_L4_nkc18_N64x1_idx-s4_octom`: one (g, tap) run spans two stages; octet-planar om (27 channels, one padded
  octet).
- `C32dg2_opp2_L2_nkc9_N64x2_idx-s8-table4x3_lrelu`: the 4x3 flow table of scale 8; a partial last slice (8 of 64).
- `C40dg5_opp1_L1_nkc12_N64x2_pre_psa_lrelu`: 45 octets, so the last stage is partial; the `pre_offset` tensor.
- `C96dg2_opp6_L1_nkc27_N64x4_idx-s2-refgw_cl`: `ref_gw != gw`, four slices (last 8), channels-last fp32 output.
- `ext_C16_opp2_L2_nkc5_N48x1_clx` and `ext_C128_opp16_L4_nkc36_N64x4`: the `_ext.dcn_v2_forward` contract (final
  offsets and mask, no sigmoid) with L = 2 and L = 4, channels-last input for the first.
- `multi_*`: B = 3 and 165 tiles, more than the 132 SMs of an H100, so CTAs run several items and the double-buffered
  flow table and the ring phases wrap mid-item: L = 1 with opp = 3 (scale 3 decode), L = 2 with nkc = 5 (not a
  multiple of the ring depth 8, scale 2 table), L = 1 at the model's large layer (C = 64, dg = 8, scale 4) and L = 4
  (scale 1 table).
Maps are ragged (H not a multiple of 16 or W not a multiple of 8) except where the id says otherwise.

The bitwise tests need no oracle: a batch equals its images run alone (other CTA counts, items per CTA and ring
phases); the flow table, the in-place decode and the materialised pyramid give identical outputs (all add the same
integer-valued floats in the same order, so any difference is a decode bug); planar and octet-planar om give
identical outputs for dg = 1, 2, 8."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


def _tiles(B, H, W):
    return B * ((H + 15) // 16) * ((W + 7) // 8)


def _geom(C, Cout, dg):
    """(opp, L, nkc, N, slices) as the host code of c2m_dcn_v2_fused_tc derives them."""
    opp = C // dg // 8
    L = min(opp, 4) if opp & (opp - 1) == 0 else 1
    nkc = (C // 8 * 9 + 3) // 4
    N = (Cout + 15) // 16 * 16 if Cout <= 64 else 64
    return opp, L, nkc, N, (Cout + 63) // 64


# (tag, B, C, Cout, dg, H, W, src, scale, ref_gw, om layout, outputs, lrelu, bias)
#   src: 'none' (om only), 'idx' (index map + scale), 'pre' (pre_offset tensor), 'ext' (_ext.dcn_v2_forward)
#   ref_gw: None = gw; outputs: 'f32', 'psa' (PSA + fp32), 'cl' (channels-last fp32), 'clx' (channels-last input)
CASES = [
    ('om-only_nobias', 1, 8, 16, 1, 5, 3, 'none', 0, None, 'planar', 'f32', False, False),
    ('idx-s1-table', 2, 24, 20, 1, 13, 15, 'idx', 1, None, 'planar', 'f32', False, True),
    ('idx-s3-decode_psa', 1, 48, 40, 2, 21, 18, 'idx', 3, None, 'planar', 'psa', False, True),
    ('idx-s4_octom', 1, 64, 64, 1, 20, 28, 'idx', 4, None, 'octet', 'f32', False, True),
    ('idx-s8-table4x3_lrelu', 2, 32, 72, 2, 24, 32, 'idx', 8, None, 'planar', 'f32', True, True),
    ('pre_psa_lrelu', 1, 40, 100, 5, 19, 13, 'pre', 1, None, 'planar', 'psa', True, True),
    ('idx-s2-refgw_cl', 1, 96, 200, 2, 18, 22, 'idx', 2, 12, 'planar', 'cl', False, True),
    ('ext_clx', 1, 16, 48, 1, 21, 13, 'ext', 0, None, 'planar', 'clx', False, True),
    ('ext', 1, 128, 256, 1, 18, 11, 'ext', 0, None, 'planar', 'f32', False, True),
    # several items per CTA (165 tiles > 132 SMs)
    ('multi_idx-s3-decode', 3, 24, 32, 1, 66, 87, 'idx', 3, None, 'planar', 'f32', False, True),
    ('multi_idx-s2-table', 3, 16, 48, 1, 66, 88, 'idx', 2, None, 'planar', 'f32', True, True),
    ('multi_model-large_idx-s4', 3, 64, 64, 8, 68, 88, 'idx', 4, None, 'octet', 'psa', True, True),
    ('multi_idx-s1-table', 3, 32, 32, 1, 66, 88, 'idx', 1, None, 'planar', 'f32', False, True),
]


def _case_id(c):
    tag, B, C, Cout, dg, H, W = c[:7]
    opp, L, nkc, N, ns = _geom(C, Cout, dg)
    head = 'ext_' if tag.startswith('ext') else 'multi_' if tag.startswith('multi') else ''
    tail = tag[len(head):]
    return (f'{head}C{C}{f"dg{dg}" if dg > 1 else ""}_opp{opp}_L{L}_nkc{nkc}_N{N}x{ns}'
            f'{"_" + tail if tail else ""}_B{B}_{H}x{W}_t{_tiles(B, H, W)}')


def _index_map(seed, B, H, W, s, ref_gw):
    """Random index map whose pyramid covers an H x W map at scale s (H = s (gh + 2)); Ref grid (gh + 1) x ref_gw."""
    gh, gw = H // s - 2, W // s - 2
    assert s * (gh + 2) == H and s * (gw + 2) == W
    rgw = ref_gw or gw
    return torch.from_numpy(np.random.default_rng(seed).integers(0, (gh + 1) * rgw, (B, gh, gw)))


def _final_offsets(om, pre, dg):
    """om[:, :2n] + the (x, y) pyramid reordered to the (h, w) pairs of the DCN offset layout."""
    n = dg * 9
    off = om[:, :2 * n].clone()
    if pre is not None:
        pr = pre.repeat(1, dg, 1, 1, 1)
        off[:, 0::2] += pr[..., 1]
        off[:, 1::2] += pr[..., 0]
    return off


def _octet_planar(om):
    from c2m_b200 import ops
    B, c, H, W = om.shape
    c8 = (c + 7) // 8
    padded = torch.zeros(B, c8 * 8, H, W, device=om.device)
    padded[:, :c] = om
    oct_om = ops.OctF32(padded.view(B, c8, 8, H, W).permute(0, 1, 3, 4, 2).contiguous(), c)
    assert torch.equal(oct_om.nchw(), om)
    return oct_om


@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_dcn_tc_edges_vs_fp64(case):
    import _ext
    from c2m_b200 import ops
    tag, B, C, Cout, dg, H, W, src, s, ref_gw, layout, outs, lrelu, has_bias = case
    assert ops.dcn_tc_supported(C, Cout, dg)
    x = seeding.randn(71, (B, C, H, W))
    wgt = seeding.randn(72, (Cout, C, 3, 3), 0.1)
    bias = seeding.randn(73, (Cout,)) if has_bias else None
    bias_or_zero = bias if has_bias else torch.zeros(Cout)
    if src == 'ext':
        off = seeding.randn(74, (B, 18 * dg, H, W), 2.0)
        off[:, :, ::2, ::3] = off[:, :, ::2, ::3].round()          # exact corners and borders
        mask = torch.sigmoid(seeding.randn(75, (B, 9 * dg, H, W)))
        want = c_oracle.dcn_v2_forward(x, wgt, bias_or_zero, off, mask, dg=dg, acc64=True)
        xd = x.to(DEV)
        if outs == 'clx':
            xd = xd.contiguous(memory_format=torch.channels_last)
        got = _ext.dcn_v2_forward(xd, wgt.to(DEV), bias.to(DEV), off.to(DEV), mask.to(DEV), 3, 3, 1, 1, 1, 1, 1, 1, dg)
        err = float((got.cpu().double() - want.double()).abs().max())
        assert err <= 2e-5 * float(want.abs().max()), err
        return
    om = seeding.randn(74, (B, 27 * dg, H, W), 0.7)
    kw = {}
    pre = None
    if src in ('idx', 'pre'):
        idx = _index_map(75, B, H, W, s, ref_gw)
        pre = torch.stack([c_oracle.offset_pyramid(idx[b], s, ref_gw) for b in range(B)])
        if src == 'idx':
            kw = dict(idx=idx.to(DEV), pre_scale=s, ref_gw=ref_gw)
        else:
            kw = dict(pre_offset=pre.to(DEV))
    want = c_oracle.dcn_v2_forward(x, wgt, bias_or_zero, _final_offsets(om, pre, dg),
                                   torch.sigmoid(om[:, 18 * dg:]), dg=dg, acc64=True)
    if lrelu:
        want = F.leaky_relu(want, 0.1)
    omd = om.to(DEV)
    if layout == 'octet':
        omd = _octet_planar(omd)
    res = ops.dcn_v2_fused_tc(x.to(DEV), omd, wgt.to(DEV), bias.to(DEV) if has_bias else None, dg, lrelu=lrelu,
                              psa_out=outs == 'psa', channels_last_out=outs == 'cl', **kw)
    gp, gf = res if outs == 'psa' else (None, res)
    if outs == 'cl':
        assert gf.is_contiguous(memory_format=torch.channels_last)
    scale = float(want.abs().max())
    err = float((gf.cpu().double() - want.double()).abs().max())
    assert err <= 2e-5 * scale, err
    if gp is not None:
        assert float((ops.psa_to_f32(gp) - gf).abs().max()) <= 1e-6 * scale


def _fused(x, om, wgt, bias, dg, **kw):
    from c2m_b200 import ops
    return ops.dcn_v2_fused_tc(x, om, wgt, bias, dg, **kw)


MULTI = [c for c in CASES if c[0].startswith('multi')]


@pytest.mark.parametrize('case', MULTI, ids=_case_id)
def test_dcn_tc_batch_invariance_bitwise(case):
    """Running an image alone changes the CTA count, the items per CTA and the ring phases, and must not change a bit."""
    tag, B, C, Cout, dg, H, W, src, s, ref_gw, layout, outs, lrelu, has_bias = case
    x = seeding.randn(81, (B, C, H, W)).to(DEV)
    om = seeding.randn(82, (B, 27 * dg, H, W), 0.7).to(DEV)
    wgt = seeding.randn(83, (Cout, C, 3, 3), 0.1).to(DEV)
    bias = seeding.randn(84, (Cout,)).to(DEV)
    idx = _index_map(85, B, H, W, s, ref_gw).to(DEV)
    full = _fused(x, om, wgt, bias, dg, idx=idx, pre_scale=s, lrelu=lrelu)
    assert torch.equal(full, _fused(x, om, wgt, bias, dg, idx=idx, pre_scale=s, lrelu=lrelu))
    for i in range(B):
        one = _fused(x[i:i + 1], om[i:i + 1], wgt, bias, dg, idx=idx[i:i + 1], pre_scale=s, lrelu=lrelu)
        assert torch.equal(full[i:i + 1], one), i


# (scale, C, dg, gh, gw, ref_gw): table scales 1, 2, 4, 8; in-place decode 3, 5; ref_gw != gw on both paths
SOURCES = [(1, 16, 2, 13, 9, None), (2, 24, 1, 9, 6, 11), (4, 32, 4, 4, 5, None), (8, 16, 1, 2, 2, 7),
           (3, 24, 1, 5, 4, None), (5, 16, 2, 3, 3, 9)]


@pytest.mark.parametrize('src', SOURCES, ids=lambda c: f's{c[0]}_{"table" if c[0] in (1, 2, 4, 8) else "decode"}'
                                                      f'_C{c[1]}dg{c[2]}{"_refgw" if c[5] else ""}')
def test_dcn_tc_offset_sources_bitwise(src):
    """The flow table, the in-place decode and the materialised pyramid add the same integer-valued floats."""
    from c2m_b200 import ops
    s, C, dg, gh, gw, ref_gw = src
    B, H, W = 2, s * (gh + 2), s * (gw + 2)
    idx = _index_map(91 + s, B, H, W, s, ref_gw)
    x = seeding.randn(92, (B, C, H, W)).to(DEV)
    om = seeding.randn(93, (B, 27 * dg, H, W), 0.7).to(DEV)
    wgt = seeding.randn(94, (40, C, 3, 3), 0.1).to(DEV)
    bias = seeding.randn(95, (40,)).to(DEV)
    pre = ops.offset_pyramid(idx.to(DEV), s, ref_gw)
    assert torch.equal(pre.cpu(), torch.stack([c_oracle.offset_pyramid(idx[b], s, ref_gw) for b in range(B)]))
    a = _fused(x, om, wgt, bias, dg, idx=idx.to(DEV), pre_scale=s, ref_gw=ref_gw)
    b = _fused(x, om, wgt, bias, dg, pre_offset=pre)
    assert torch.equal(a, b)


@pytest.mark.parametrize('dg', [1, 2, 8])
def test_dcn_tc_om_layout_bitwise(dg):
    """Planar and octet-planar om (27 dg channels, padded to whole octets for dg = 1, 2) give identical outputs."""
    B, C, H, W, s = 2, 64, 30, 22, 2
    idx = _index_map(101, B, H, W, s, None).to(DEV)
    x = seeding.randn(102, (B, C, H, W)).to(DEV)
    om = seeding.randn(103, (B, 27 * dg, H, W), 0.7).to(DEV)
    wgt = seeding.randn(104, (64, C, 3, 3), 0.1).to(DEV)
    bias = seeding.randn(105, (64,)).to(DEV)
    a = _fused(x, om, wgt, bias, dg, idx=idx, pre_scale=s)
    b = _fused(x, _octet_planar(om), wgt, bias, dg, idx=idx, pre_scale=s)
    assert torch.equal(a, b)
