"""Correlation search (`corr_umma_kernel` + rescoring, csrc/corr_umma.cu, csrc/corr_aux.cu) at its untested
configurations (-m gpu).

The wgmma search takes every patch-3, stride-1 call whose maps are at least 10x16 on both sides.  It tiles the query
patch grid into 8 x 14 blocks and the Ref patch grid likewise, streams 4 channel octets per K stage, and splits the
Ref tiles of each query tile into `nchunk` chunks (`corr_umma_pick_nchunk`, mirrored by `_pick_nchunk` below); the
last chunk may be shorter.  A work item is (image, query tile, chunk); with more items than SMs a CTA takes several.
The rescoring pass then makes the index map exact: a query may differ from the fp64 oracle only where its top-1 /
top-2 gap is below 1e-6 of that query's score scale, and `force_generic=True` (the CUDA-core search) must return the
same idx and val bit for bit.

Case ids name the C, batch, map sizes, tile counts, chunking (`ch<n>` / `ch<n>short` when the last chunk is short)
and items (`_over_sms` when CTAs run several).  What each case pins:
- `min_C8`: the minimum wgmma maps (10x16 both sides), one octet (K stage mostly TMA zero fill).
- `c20`: C = 20 (padded to 24 = 3 octets by the prep), B = 2, Ref 13x30.
- `c40_raw`: gw = 28 (two full 14-wide tiles) against rw = 29 (one past), `is_norm=False`, C = 40 (5 octets).
- `c96`: gh = 24, gw = 42 (whole tiles) against a Ref one larger on each side, `norm_input=False`, C = 96 (3 stages).
- `c256_b3_chunks`: several Ref chunks with a short last one, B = 3.
- `c64_b4`: 64x64 maps, B = 4: more items than SMs (the oracle checks the last image's ragged last query-tile row).
- `below_10x15`: one column short of the threshold, so the generic search runs; it must give the same answer.
Each runs with `l2norm` off and on (on: checked against `F.normalize` + the oracle).

Dynamic range (`dyn_*`): the prep scales each map by one power of two chosen from its largest |x| over the whole
batch, so elements far below it fall into the fp16 subnormals, where the rounding error of the operands is absolute
rather than relative.  A query map at 1e-7 / 1e-8 with one element at 1.0, a Ref map at 1e-5 / 1e-6 with one
element at 1e3, and a batch whose second image is the first times 1e-8 must still give the exact argmax.

A batch equals its images run alone under C2M_CORR_EXACT_TIES=1 (exact mode: always the exhaustive answer; in the
default mode the overflow budget depends on the number of queries of the call)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


def _cdiv(a, b):
    return -(-a // b)


def _wgmma(h, w, hr, wr):
    """corr_umma_supported for patch 3, stride 1."""
    return w >= 16 and h >= 10 and wr >= 16 and hr >= 10


def _tiles(gh, gw, rh, rw):
    """corr_umma_tiles: 8-row x 14-column blocks of patch origins on both sides."""
    return _cdiv(gh, 8) * _cdiv(gw, 14), _cdiv(rh, 8) * _cdiv(rw, 14)


def _pick_nchunk(B, gh, gw, rh, rw, sms):
    """Mirror of corr_umma_pick_nchunk (corr_umma.cu): the split minimising waves x (tiles per item + 0.35) plus the
    re-scan allowance, with no empty chunks."""
    n_qt, n_rt = _tiles(gh, gw, rh, rw)
    best_n, best_cost = 1, 1e300
    for n in range(1, min(32, n_rt) + 1):
        per = _cdiv(n_rt, n)
        if _cdiv(n_rt, per) != n:
            continue
        waves = _cdiv(B * n_qt * n, sms)
        cost = waves * (per + 0.35) + B * n_qt * 2e-3 * per
        if cost < best_cost - 1e-9:
            best_cost, best_n = cost, n
    return best_n


def _chunking(case):
    """(n_qt, n_rt, nchunk, short last chunk, items) of a case on this device."""
    _, B, C, h, w, hr, wr = case[:7]
    gh, gw, rh, rw = h - 2, w - 2, hr - 2, wr - 2
    n_qt, n_rt = _tiles(gh, gw, rh, rw)
    n = _pick_nchunk(B, gh, gw, rh, rw, SMS)
    per = _cdiv(n_rt, n)
    return n_qt, n_rt, n, n_rt - (n - 1) * per < per, B * n_qt * n


# (tag, B, C, h, w, hr, wr, is_norm, norm_input)
CASES = [
    ('min_C8', 1, 8, 10, 16, 10, 16, True, True),
    ('c20', 2, 20, 12, 20, 13, 30, True, True),
    ('c40_raw', 1, 40, 12, 30, 14, 31, False, False),
    ('c96', 1, 96, 26, 44, 27, 45, True, False),
    ('c256_b3_chunks', 3, 256, 12, 32, 19, 31, True, True),
    ('c64_b4', 4, 64, 64, 64, 64, 64, True, True),
    ('below_10x15', 1, 32, 10, 15, 12, 18, True, True),
]


def _case_id(c):
    tag, B, C, h, w, hr, wr = c[:7]
    if not _wgmma(h, w, hr, wr):
        return f'{tag}_B{B}_{h}x{w}_vs_{hr}x{wr}_generic'
    n_qt, n_rt, n, short, items = _chunking(c)
    return (f'{tag}_B{B}_{h}x{w}_vs_{hr}x{wr}_qt{n_qt}_rt{n_rt}_ch{n}{"short" if short else ""}'
            f'_items{items}{"_over_sms" if items > SMS else ""}')


def test_corr_case_table_covers_chunking():
    wg = [c for c in CASES if _wgmma(*c[3:7])]
    assert any(_chunking(c)[3] for c in wg), 'no case with a short last Ref chunk'
    assert any(_chunking(c)[4] > SMS for c in wg), 'no case with more work items than SMs'
    assert any(not _wgmma(*c[3:7]) for c in CASES)


def _patch_norms(f):
    """fp64 norm of every 3x3 patch of a [C, h, w] map, as a [h-2, w-2] tensor."""
    C, h, w = f.shape
    return F.unfold(f[None].double(), 3).norm(dim=1).view(h - 2, w - 2)


def _check_vs_oracle(idx, val, fin, fref, is_norm, norm_input, rows=None):
    """idx / val of one image against the fp64 oracle.  A differing query is tolerated only where the oracle's top-1 /
    top-2 gap is below 1e-6 of the query's score scale (||P_q||, times the largest Ref patch norm for raw scores).
    rows: (r0, r1) restricts the check to query rows [r0, r1) (the oracle then sees only those rows of the map)."""
    r0, r1 = rows or (0, idx.shape[0])
    fq = fin[:, r0:r1 + 2]
    want_i, want_v, gap = c_oracle.corr_argmax(fq, fref, is_norm=is_norm, norm_input=norm_input, want_gap=True)
    idx, val = idx[r0:r1].cpu(), val[r0:r1].cpu()
    scale = _patch_norms(fq) * (1.0 if is_norm else float(_patch_norms(fref).max()))
    bad = idx != want_i
    assert int(bad.sum()) == 0 or bool((gap[bad] < 1e-6 * scale[bad]).all()), \
        (int(bad.sum()), float((gap[bad] / scale[bad]).max()))
    ok = ~bad.numpy()
    vs = float(want_v.abs().max())
    np.testing.assert_allclose(val.numpy()[ok], want_v.numpy()[ok], rtol=1e-5, atol=1e-6 * vs)


def _run_and_check(fin, fref, is_norm, norm_input, l2norm, rows=None, images=None):
    import c2m_b200 as c2m
    fd, rd = fin.to(DEV), fref.to(DEV)
    kw = dict(is_norm=is_norm, norm_input=norm_input, l2norm=l2norm)
    idx, val = c2m.corr_argmax(fd, rd, **kw)
    idx_g, val_g = c2m.corr_argmax(fd, rd, force_generic=True, **kw)
    assert torch.equal(idx, idx_g) and torch.equal(val, val_g), int((idx != idx_g).sum())
    B = fin.shape[0]
    for b in (range(B) if images is None else images):
        a, r = fin[b], fref[b]
        if l2norm:
            a, r = F.normalize(a, dim=0), F.normalize(r, dim=0)
        _check_vs_oracle(idx[b], val[b], a, r, is_norm, norm_input, rows)
    return idx, val


def _inputs(case):
    tag, B, C, h, w, hr, wr = case[:7]
    return seeding.randn(201, (B, C, h, w)), seeding.randn(202, (B, C, hr, wr))


@pytest.mark.parametrize('l2norm', [False, True], ids=['raw', 'l2norm'])
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_corr_edges_vs_fp64(case, l2norm):
    import c2m_b200 as c2m
    tag, B, C, h, w, hr, wr, is_norm, norm_input = case
    fin, fref = _inputs(case)
    big = B * (h - 2) * (w - 2) * (hr - 2) * (wr - 2) > 5e7
    # large maps: the oracle checks the last image's last 8 query rows (a partial query tile for 64x64)
    idx, val = _run_and_check(fin, fref, is_norm, norm_input, l2norm, rows=(h - 10, h - 2) if big else None,
                              images=[B - 1] if big else None)
    if B == 1 and not l2norm:
        idx1, val1 = c2m.feature_match_index(fin[0].to(DEV), fref[0].to(DEV), 3, 1, 1, is_norm, norm_input)
        assert torch.equal(idx1, idx[0]) and torch.equal(val1, val[0])


@pytest.mark.parametrize('l2norm', [False, True], ids=['raw', 'l2norm'])
@pytest.mark.parametrize('case', [c for c in CASES if c[1] > 1], ids=_case_id)
def test_corr_edges_batch_invariance_exact_mode(case, l2norm, monkeypatch):
    import c2m_b200 as c2m
    monkeypatch.setenv('C2M_CORR_EXACT_TIES', '1')
    tag, B, C, h, w, hr, wr, is_norm, norm_input = case
    fin, fref = [t.to(DEV) for t in _inputs(case)]
    kw = dict(is_norm=is_norm, norm_input=norm_input, l2norm=l2norm)
    idx, val = c2m.corr_argmax(fin, fref, **kw)
    for b in range(B):
        i1, v1 = c2m.corr_argmax(fin[b:b + 1], fref[b:b + 1], **kw)
        assert torch.equal(i1, idx[b:b + 1]) and torch.equal(v1, val[b:b + 1]), b


def _dyn_inputs(tag):
    """C = 64, query map 20x22 (18x20 patches), Ref map 24x26 (22x24 patches), per-pixel unit features."""
    fin = seeding.unit_features(211, 64, 20, 22)
    fref = seeding.unit_features(212, 64, 24, 26)
    if tag == 'q1e-7' or tag == 'q1e-8':
        fin = fin * (1e-7 if tag == 'q1e-7' else 1e-8)
        fin[5, 3, 4] = 1.0
    elif tag == 'r1e-5' or tag == 'r1e-6':
        fref = fref * (1e-5 if tag == 'r1e-5' else 1e-6)
        fref[7, 10, 12] = 1e3
    elif tag == 'batch1e-8':
        return torch.stack([fin, fin * 1e-8]), torch.stack([fref, fref * 1e-8])
    return fin[None], fref[None]


@pytest.mark.parametrize('tag', ['q1e-7', 'q1e-8', 'r1e-5', 'r1e-6', 'batch1e-8'])
def test_corr_dynamic_range_vs_fp64(tag):
    """Elements far below the map's (batch's) largest one land in the fp16 subnormals of the split operands; the
    rescoring window must cover their absolute rounding error, or the exact winner is never rescored."""
    fin, fref = _dyn_inputs(tag)
    _run_and_check(fin, fref, True, True, False)
