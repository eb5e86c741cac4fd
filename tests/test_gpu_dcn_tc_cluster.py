"""Tensor-core DCN with more than 64 output channels (-m gpu): one cluster launch, bit-identical to its slices.

When Cout > 64, `c2m_dcn_v2_fused_tc` launches `dcn_wgmma_kernel` in thread-block clusters of S = ceil(Cout / 64)
CTAs.  CTA r of a cluster computes output channels [64 r, 64 r + 64) of the cluster's tiles, and the gathered column
stages are built once per cluster: ring slot i is filled by CTA i % S and bulk-copied into the other CTAs.  Each
slice's arithmetic is that of a Cout <= 64 launch, so a layer must equal, bit for bit, its 64-row slices computed one
by one as separate Cout <= 64 calls with the matching weight and bias rows.  The weight pack takes one scale exponent
from the largest |w| of the whole tensor, so every 64-row slice is given the same largest |w|.

Each case id names: C/dg, L (K octets per gather thread; L stage groups work on L of the CTA's stages at once), nkc
(K stages, here not always a multiple of S), the cluster size S, the offset source and the outputs, the batch, the map and the item (tile) count.  The item counts
cover fewer items than an H100 has clusters and counts that are not a multiple of the cluster count (CTAs of one
cluster then run several items and the ring phases wrap mid-item)."""
import numpy as np
import pytest
import torch

import seeding

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


# (tag, B, C, Cout, dg, H, W, src, scale, om layout, outputs, lrelu, bias)
#   src: 'idx' (index map + scale), 'pre' (pre_offset tensor), 'ext' (final offsets and mask, fp32 input)
#   outputs: 'f32' or 'psa' (PSA + fp32)
CASES = [
    ('idx-s1_octom_psa', 1, 72, 128, 9, 37, 29, 'idx', 1, 'octet', 'psa', True, True),
    ('idx-s2', 5, 64, 256, 8, 34, 22, 'idx', 2, 'planar', 'f32', False, True),
    ('idx-s4_octom_psa', 2, 128, 160, 8, 44, 36, 'idx', 4, 'octet', 'psa', True, True),
    ('idx-s3-decode', 1, 48, 160, 2, 21, 18, 'idx', 3, 'planar', 'f32', False, True),
    ('idx-s4_cout72', 1, 72, 72, 9, 20, 28, 'idx', 4, 'planar', 'f32', True, True),
    ('pre_nobias', 1, 40, 100, 5, 19, 13, 'pre', 1, 'planar', 'psa', False, False),
    ('ext', 2, 128, 256, 1, 18, 11, 'ext', 0, 'planar', 'f32', False, True),
    ('ext_dg8', 5, 64, 128, 8, 23, 17, 'ext', 0, 'planar', 'f32', False, True),
    ('ext_dg8', 1, 256, 128, 8, 20, 12, 'ext', 0, 'planar', 'f32', True, True),
    # the model's small and medium layers: more items than clusters, not a multiple of the cluster count
    ('model-small_idx-s1_octom_psa', 5, 256, 256, 8, 40, 40, 'idx', 1, 'octet', 'psa', True, True),
    ('model-medium_idx-s2', 3, 128, 128, 8, 66, 88, 'idx', 2, 'planar', 'f32', True, True),
]


def _geom(C, Cout, dg):
    """(L, nkc, S) as the host code derives them: a cluster of S CTAs has a ring of 8 stages (6 when S = 3) and keeps
    L * S within it."""
    opp = C // dg // 8
    L = min(opp, 4) if opp & (opp - 1) == 0 else 1
    S = (Cout + 63) // 64
    return min(L, (6 if S == 3 else 8) // S), (C // 8 * 9 + 3) // 4, S


def _case_id(c):
    tag, B, C, Cout, dg, H, W = c[:7]
    L, nkc, S = _geom(C, Cout, dg)
    tiles = B * ((H + 15) // 16) * ((W + 7) // 8)
    return f'C{C}{f"dg{dg}" if dg > 1 else ""}_L{L}_nkc{nkc}_S{S}_{tag}_B{B}_{H}x{W}_t{tiles}'


def _index_map(seed, B, H, W, s):
    gh, gw = H // s - 2, W // s - 2
    assert s * (gh + 2) == H and s * (gw + 2) == W
    return torch.from_numpy(np.random.default_rng(seed).integers(0, (gh + 1) * gw, (B, gh, gw)))


def _octet_planar(om):
    from c2m_b200 import ops
    B, c, H, W = om.shape
    c8 = (c + 7) // 8
    padded = torch.zeros(B, c8 * 8, H, W, device=om.device)
    padded[:, :c] = om
    return ops.OctF32(padded.view(B, c8, 8, H, W).permute(0, 1, 3, 4, 2).contiguous(), c)


@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_dcn_tc_cluster_equals_slices(case):
    from c2m_b200 import ops
    tag, B, C, Cout, dg, H, W, src, s, layout, outs, lrelu, has_bias = case
    assert ops.dcn_tc_supported(C, Cout, dg) and Cout > 64
    x = seeding.randn(91, (B, C, H, W)).to(DEV)
    wgt = seeding.randn(92, (Cout, C, 3, 3), 0.1)
    for r in range(0, Cout, 64):
        wgt[r, r // 64 % C, 1, 1] = 1.0          # the same largest |w| in every slice
    wgt = wgt.to(DEV)
    bias = seeding.randn(93, (Cout,)).to(DEV) if has_bias else None
    kw = dict(lrelu=lrelu, psa_out=outs == 'psa')
    if src == 'ext':
        om = seeding.randn(94, (B, 18 * dg, H, W), 2.0).to(DEV)
        kw['final_mask'] = torch.sigmoid(seeding.randn(95, (B, 9 * dg, H, W))).to(DEV)
    else:
        om = seeding.randn(94, (B, 27 * dg, H, W), 0.7).to(DEV)
        if layout == 'octet':
            om = _octet_planar(om)
        if src == 'idx':
            kw.update(idx=_index_map(95, B, H, W, s).to(DEV), pre_scale=s)
        else:
            kw['pre_offset'] = seeding.randn(95, (B, 9, H, W, 2), 3.0).to(DEV)
        xp = ops.psa_from_f32(x)
        x = xp                                   # the model's PSA input

    def run(w, b):
        res = ops.dcn_v2_fused_tc(x, om, w, b, dg, **kw)
        return res if outs == 'psa' else (None, res)

    full_p, full_f = run(wgt, bias)
    again_p, again_f = run(wgt, bias)
    assert torch.equal(full_f, again_f)
    if full_p is not None:
        assert torch.equal(full_p.hi, again_p.hi) and torch.equal(full_p.lo, again_p.lo)
    for r in range(0, Cout, 64):
        n = min(64, Cout - r)
        part_p, part_f = run(wgt[r:r + n].contiguous(), bias[r:r + n].contiguous() if has_bias else None)
        assert torch.equal(full_f[:, r:r + n], part_f), f'slice {r // 64}'
        if full_p is not None:
            o = r // 8
            assert torch.equal(full_p.hi[:, o:o + part_p.hi.shape[1]], part_p.hi), f'slice {r // 64} (PSA hi)'
            assert torch.equal(full_p.lo[:, o:o + part_p.lo.shape[1]], part_p.lo), f'slice {r // 64} (PSA lo)'
