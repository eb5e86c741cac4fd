"""The correlation oracle (`oracle_corr_argmax`, oracle/c2m_oracle.c) on non-finite inputs, checked on the CPU.

The reference (`feature_match_index`: F.conv2d of the query map with the normalised Ref patches, then `max(dim=0)`)
follows torch's `max` rule: a NaN score is the maximum, the first NaN Ref patch wins and val is NaN; +Inf is an
ordinary maximum, ties to the lowest index.  Under `is_norm` a Ref patch holding an Inf has norm Inf and scores NaN
(Inf / Inf).  The oracle is pinned here against `oracle/ref_path.feature_match_index` run in fp64 on maps small enough
for one Ref chunk: val's finiteness pattern must be equal, idx must be equal on every non-finite query, and on the
finite ones it may differ only where the oracle's top-1 / top-2 gap is below 1e-6 of the query's score scale (the
oracle normalises the Ref patches in fp32, ref_path in fp64)."""
import math

import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle, ref_path

C, H, W, HR, WR = 5, 6, 7, 7, 8


@pytest.fixture(scope='module', autouse=True)
def _oracle_built():
    c_oracle.build()


def _patch_norms(f):
    C_, h, w = f.shape
    return F.unfold(f[None].double(), 3).norm(dim=1).view(h - 2, w - 2)


def _check(fin, fref, is_norm, norm_input):
    want_i, want_v = ref_path.feature_match_index(fin.double(), fref.double(), 3, 1, 1, is_norm, norm_input)
    got_i, got_v, gap = c_oracle.corr_argmax(fin, fref, is_norm=is_norm, norm_input=norm_input, want_gap=True)
    fin_w, fin_g = torch.isfinite(want_v), torch.isfinite(got_v)
    assert torch.equal(fin_w, fin_g), (want_v, got_v)
    nf = ~fin_w
    assert torch.equal(torch.isnan(want_v[nf]), torch.isnan(got_v[nf]))
    assert torch.equal(want_v[nf & ~torch.isnan(want_v)].float(), got_v[nf & ~torch.isnan(got_v)])
    assert torch.equal(want_i[nf], got_i[nf]), (want_i, got_i)
    fq = torch.nan_to_num(fin, 0.0, 0.0, 0.0)
    fr = torch.nan_to_num(fref, 0.0, 0.0, 0.0)
    pr = _patch_norms(fr)
    scale = _patch_norms(fq) * float((pr / (pr + 1e-5)).max() if is_norm else pr.max())
    bad = fin_w & (want_i != got_i)
    assert bool((gap[bad] < 1e-6 * scale[bad]).all()), int(bad.sum())
    if bool(fin_w.any()):        # val on every finite query; one that took the other side of a tie by up to its gap
        w, g = want_v[fin_w], got_v[fin_w].double()
        qdiv = (_patch_norms(fq)[fin_w] + 1e-5) if norm_input else 1.0
        bar = 1e-5 * w.abs() + 1e-6 * float(w.abs().max()) + torch.where(bad[fin_w], gap[fin_w], 0.0) / qdiv
        assert bool(((g - w).abs() <= bar).all()), float(((g - w).abs() / bar).max())
    return got_i, got_v


def _spots(h, w):
    return {'corner00': (0, 0), 'corner_last': (h - 1, w - 1), 'border': (0, w // 2), 'inside': (h // 2, w // 2)}


@pytest.mark.parametrize('is_norm', [True, False], ids=['is_norm', 'raw'])
@pytest.mark.parametrize('value', [math.nan, math.inf, -math.inf], ids=['nan', 'pinf', 'ninf'])
@pytest.mark.parametrize('spot', ['corner00', 'corner_last', 'border', 'inside'])
@pytest.mark.parametrize('where', ['query', 'ref'])
def test_oracle_nonfinite_vs_reference_fp64(where, spot, value, is_norm):
    fin = seeding.randn(301, (C, H, W))
    fref = seeding.randn(302, (C, HR, WR))
    t = fin if where == 'query' else fref
    y, x = _spots(t.shape[1], t.shape[2])[spot]
    t[1, y, x] = value
    t[3, y, x] = 100.0
    _check(fin, fref, is_norm, is_norm)


@pytest.mark.parametrize('is_norm', [True, False], ids=['is_norm', 'raw'])
def test_oracle_nonfinite_row_and_zero_region(is_norm):
    """A whole NaN row in the Ref map, an Inf and a zero region in the query map."""
    fin = seeding.randn(303, (C, H, W))
    fref = seeding.randn(304, (C, HR, WR))
    fref[:, 4, :] = math.nan
    fin[:, 0:3, 0:3] = 0.0
    fin[2, 5, 6] = math.inf
    _check(fin, fref, is_norm, False)


def test_oracle_nonfinite_hand_worked():
    """Patch 1, one channel, raw scores: query values 1, -1, 0 against Ref values 2, +Inf, -Inf, 3.
    q = 1: scores (2, Inf, -Inf, 3) -> (Inf, 1); q = -1: (-2, -Inf, Inf, -3) -> (Inf, 2); q = 0: (0, NaN, NaN, 0)
    -> (NaN, 1), the first NaN."""
    fin = torch.tensor([[[1.0, -1.0, 0.0]]])
    fref = torch.tensor([[[2.0, math.inf, -math.inf, 3.0]]])
    idx, val = c_oracle.corr_argmax(fin, fref, patch=1, is_norm=False)
    assert idx.tolist() == [[1, 2, 1]]
    assert val[0, :2].tolist() == [math.inf, math.inf] and math.isnan(float(val[0, 2]))
    want_i, want_v = ref_path.feature_match_index(fin.double(), fref.double(), 1, 1, 1, False, False)
    assert torch.equal(want_i, idx)
    assert torch.equal(torch.isnan(want_v), torch.isnan(val))
