"""Correlation search (`corr_argmax` / `feature_match_index`: prep, `corr_umma_kernel` or `search_generic_kernel`, the
exact rescoring) across the fp32 range and with non-finite inputs (-m gpu).

Contract (DESIGN.md K2).  Finite inputs: idx / val equal `oracle_corr_argmax` (the reference's arithmetic with an
error-free accumulation); a query may differ only where the oracle's top-1 / top-2 gap is below 1e-6 of its score
scale, at every input magnitude where the oracle's scores are normal fp32 numbers.  Non-finite inputs follow torch's
`max` over the whole Ref set: a NaN score is the maximum (the lowest NaN Ref index wins, val NaN), +Inf is an
ordinary maximum.

Every case runs both routes, the wgmma search and `force_generic=True`, and they must agree bit for bit.  Two
geometries: C 64 with a 20x30 query map against a 26x34 Ref map (several Ref chunks, ragged tiles) and C 256 at the
10x16 minimum of the wgmma route.  C2M_CORR_EXACT_TIES=1 (always the exhaustive answer) where the answer is a tie
among many Ref patches (a map that collapses to zero)."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

# (tag, C, h, w, hr, wr)
GEOMS = [('c64_20x30_vs_26x34', 64, 20, 30, 26, 34), ('c256_10x16', 256, 10, 16, 10, 16)]
SCALES = [1e-30, 1e-20, 1e-6, 1.0, 1e6, 1e18, 1e30]
SCALES_L2 = [1e-30, 1.0, 1e30]              # l2norm: every scale in between normalises to the same maps
# (is_norm, norm_input)
NORMS = [(True, True), (True, False), (False, False)]


_WORST = {}          # test function -> largest val error over its bar, printed at the end of the module (-s)


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    yield
    for name, r in sorted(_WORST.items()):
        print(f'\n{name}: largest val error / bar = {r:.3f}')


def _geom_id(g):
    return g[0]


def _norm_id(n):
    return {(True, True): 'norm_in', (True, False): 'norm', (False, False): 'raw'}[n]


def _inputs(geom, seed, B=1):
    _, C, h, w, hr, wr = geom
    return seeding.randn(seed, (B, C, h, w)), seeding.randn(seed + 1, (B, C, hr, wr))


def _patch_norms(f):
    """fp64 norm of every 3x3 patch of a [C, h, w] map (non-finite elements counted as 0), as [h-2, w-2]."""
    C, h, w = f.shape
    f = torch.nan_to_num(f.double(), 0.0, 0.0, 0.0)
    return F.unfold(f[None], 3).norm(dim=1).view(h - 2, w - 2)


def _score_scales(fin, fref, is_norm):
    """Per query, the largest |score| it can have (fp64): ||P_q|| max_r ||P_r|| / (||P_r|| + 1e-5), or
    ||P_q|| max_r ||P_r|| for raw scores.  Under is_norm a Ref map far below 1e-5 scales every score down with it."""
    pr = _patch_norms(fref)
    return _patch_norms(fin) * float((pr / (pr + 1e-5)).max() if is_norm else pr.max())


def _bits(v):
    return v.contiguous().view(torch.int32)


def _run(fin, fref, is_norm, norm_input, l2norm):
    """Both routes on the GPU; they must agree bit for bit (NaN included)."""
    import c2m_b200 as c2m
    fd, rd = fin.to(DEV), fref.to(DEV)
    kw = dict(is_norm=is_norm, norm_input=norm_input, l2norm=l2norm)
    idx, val = c2m.corr_argmax(fd, rd, **kw)
    idx_g, val_g = c2m.corr_argmax(fd, rd, force_generic=True, **kw)
    assert torch.equal(idx, idx_g), int((idx != idx_g).sum())
    assert torch.equal(_bits(val), _bits(val_g)), int((_bits(val) != _bits(val_g)).sum())
    return idx.cpu(), val.cpu()


def _check(idx, val, fin, fref, is_norm, norm_input, l2norm):
    """One image against the oracle (run on F.normalize's output when l2norm).  val's finiteness pattern is the
    oracle's; non-finite queries have the oracle's idx and val class (NaN / +-Inf); a finite query's idx may differ
    only under the gap rule, and its val is the oracle's to 1e-5.  Returns the largest val error over its bar."""
    if l2norm:
        fin, fref = F.normalize(fin, dim=0), F.normalize(fref, dim=0)
    want_i, want_v, gap = c_oracle.corr_argmax(fin, fref, is_norm=is_norm, norm_input=norm_input, want_gap=True)
    fw = torch.isfinite(want_v)
    diff = fw != torch.isfinite(val)
    assert not bool(diff.any()), (int(diff.sum()), want_v[diff][:4], val[diff][:4])
    nf = ~fw
    assert torch.equal(idx[nf], want_i[nf]), int((idx[nf] != want_i[nf]).sum())
    assert torch.equal(torch.isnan(val[nf]), torch.isnan(want_v[nf]))
    assert torch.equal(val[nf & ~torch.isnan(val)], want_v[nf & ~torch.isnan(want_v)])
    scale = _score_scales(fin, fref, is_norm)
    bad = fw & (idx != want_i)
    assert bool((gap[bad] < 1e-6 * scale[bad]).all()), (int(bad.sum()), float((gap[bad] / scale[bad]).max()))
    if not bool(fw.any()):
        return 0.0
    # val on every finite query; a query that took the other side of a sub-1e-6 tie may differ by that gap too
    w64, v64 = want_v[fw].double(), val[fw].double()
    qdiv = (_patch_norms(fin)[fw] + 1e-5) if norm_input else 1.0
    bar = 1e-5 * w64.abs() + 1e-6 * float(w64.abs().max()) + torch.where(bad[fw], gap[fw], 0.0) / qdiv
    ratio = float(((v64 - w64).abs() / bar.clamp_min(torch.finfo(torch.float64).tiny)).max())   # bar 0: all scores 0
    assert ratio <= 1.0, ratio
    name = os.environ.get('PYTEST_CURRENT_TEST', '').split('::')[-1].split('[')[0]
    _WORST[name] = max(_WORST.get(name, 0.0), ratio)
    return ratio


def _score_scale(sq, sr, is_norm, K):
    """Typical magnitude of a winning score for maps of element scale sq (query) and sr (Ref)."""
    pn = sr * math.sqrt(K)
    return sq * 3.0 * (pn / (pn + 1e-5) if is_norm else sr * math.sqrt(K))


def _sweep_cases():
    out = []
    for g in GEOMS:
        K = 9 * g[1]
        for sq in SCALES:
            for sr in SCALES:
                for n in NORMS:
                    for l2 in (False, True):
                        if l2 and not (sq in SCALES_L2 and sr in SCALES_L2):
                            continue
                        s = _score_scale(sq, sr, n[0], K)
                        if not l2 and not 1e-34 <= s <= 1e33:
                            continue                            # the oracle's scores leave the normal fp32 range
                        out.append(pytest.param(g, sq, sr, n, l2, id=f'{g[0]}-q{sq:g}-r{sr:g}-{_norm_id(n)}'
                                                                       f'-{"l2norm" if l2 else "plain"}'))
    return out


@pytest.mark.parametrize('geom,sq,sr,norm,l2norm', _sweep_cases())
def test_corr_scale_sweep_vs_oracle(geom, sq, sr, norm, l2norm, monkeypatch):
    """Query map times sq, Ref map times sr: the answer is the oracle's at every scale pair whose scores are normal.
    Under l2norm a map at 1e30 normalises to zero (fp32 norm overflow, as F.normalize), and every score ties."""
    if l2norm and max(sq, sr) > 1e18:
        monkeypatch.setenv('C2M_CORR_EXACT_TIES', '1')
    fin, fref = _inputs(geom, 401)
    fin, fref = fin * sq, fref * sr
    idx, val = _run(fin, fref, *norm, l2norm)
    _check(idx[0], val[0], fin[0], fref[0], *norm, l2norm)


_BASE = {}


def _base(geom, is_norm):
    key = (geom[0], is_norm)
    if key not in _BASE:
        fin, fref = _inputs(geom, 411)
        _BASE[key] = (fin, fref, _run(fin, fref, is_norm, False, False))
    return _BASE[key]


POW = [-60, -24, -11, 11, 24, 60]


@pytest.mark.parametrize('j', POW)
@pytest.mark.parametrize('k', POW)
@pytest.mark.parametrize('geom', GEOMS, ids=_geom_id)
def test_corr_power_of_two_scaling_raw(geom, k, j):
    """is_norm=False: query times 2^k, Ref times 2^j -> idx unchanged, val exactly 2^(k+j) times."""
    fin, fref, (idx, val) = _base(geom, False)
    i2, v2 = _run(fin * 2.0 ** k, fref * 2.0 ** j, False, False, False)
    assert torch.equal(i2, idx), int((i2 != idx).sum())
    assert torch.equal(v2, val * 2.0 ** (k + j))


@pytest.mark.parametrize('k', POW)
@pytest.mark.parametrize('geom', GEOMS, ids=_geom_id)
def test_corr_power_of_two_scaling_is_norm(geom, k):
    """is_norm=True: query times 2^k -> idx unchanged, val exactly 2^k times (the Ref's + 1e-5 is not scale-free)."""
    fin, fref, (idx, val) = _base(geom, True)
    i2, v2 = _run(fin * 2.0 ** k, fref, True, False, False)
    assert torch.equal(i2, idx), int((i2 != idx).sum())
    assert torch.equal(v2, val * 2.0 ** k)


MIXED = [1.0, 1e-20, 1e20]


@pytest.mark.parametrize('l2norm', [False, True], ids=['plain', 'l2norm'])
@pytest.mark.parametrize('norm', NORMS, ids=_norm_id)
def test_corr_mixed_scale_batch(norm, l2norm, monkeypatch):
    """Images at 1, 1e-20 and 1e20 in one call (both maps; the query only for raw scores, whose product would leave
    fp32): each image against its own oracle, and equal bit for bit to the image run alone."""
    monkeypatch.setenv('C2M_CORR_EXACT_TIES', '1')
    geom = GEOMS[0]
    fin, fref = _inputs(geom, 421, B=3)
    s = torch.tensor(MIXED).view(3, 1, 1, 1)
    fin = fin * s
    fref = fref * (s if norm[0] else 1.0)
    idx, val = _run(fin, fref, *norm, l2norm)
    for b in range(3):
        _check(idx[b], val[b], fin[b], fref[b], *norm, l2norm)
        i1, v1 = _run(fin[b:b + 1], fref[b:b + 1], *norm, l2norm)
        assert torch.equal(i1[0], idx[b]) and torch.equal(_bits(v1[0]), _bits(val[b])), b


def _spots(h, w):
    return {'corner00': (0, 0), 'corner_last': (h - 1, w - 1), 'border': (h - 1, w // 2), 'inside': (h // 2, w // 3)}


NONFINITE = {'nan': math.nan, 'pinf': math.inf, 'ninf': -math.inf}


@pytest.mark.parametrize('l2norm', [False, True], ids=['plain', 'l2norm'])
@pytest.mark.parametrize('norm', [(True, True), (False, False)], ids=_norm_id)
@pytest.mark.parametrize('value', list(NONFINITE), ids=list(NONFINITE))
@pytest.mark.parametrize('spot', ['corner00', 'corner_last', 'border', 'inside'])
@pytest.mark.parametrize('where', ['query', 'ref'])
@pytest.mark.parametrize('geom', GEOMS, ids=_geom_id)
def test_corr_nonfinite_vs_oracle(geom, where, spot, value, norm, l2norm):
    """One NaN / +-Inf element, with finite elements of magnitude 100 in the same map (above fp16's range once an
    Inf sets the map's scale)."""
    fin, fref = _inputs(geom, 431)
    t = fin if where == 'query' else fref
    _, C, H, W = t.shape
    y, x = _spots(H, W)[spot]
    t[0, 1, y, x] = NONFINITE[value]
    t[0, 3, H // 2 - 1, W // 2 + 1] = 100.0
    t[0, 5, 1, W - 2] = -100.0
    idx, val = _run(fin, fref, *norm, l2norm)
    _check(idx[0], val[0], fin[0], fref[0], *norm, l2norm)


@pytest.mark.parametrize('l2norm', [False, True], ids=['plain', 'l2norm'])
@pytest.mark.parametrize('norm', [(True, True), (False, False)], ids=_norm_id)
@pytest.mark.parametrize('where', ['query', 'ref'])
@pytest.mark.parametrize('geom', GEOMS, ids=_geom_id)
def test_corr_nan_row_vs_oracle(geom, where, norm, l2norm):
    """A whole NaN image row: every query (or every Ref patch) touching it scores NaN."""
    fin, fref = _inputs(geom, 441)
    t = fin if where == 'query' else fref
    t[0, :, t.shape[2] // 2, :] = math.nan
    idx, val = _run(fin, fref, *norm, l2norm)
    _check(idx[0], val[0], fin[0], fref[0], *norm, l2norm)


@pytest.mark.parametrize('l2norm', [False, True], ids=['plain', 'l2norm'])
@pytest.mark.parametrize('norm', NORMS, ids=_norm_id)
@pytest.mark.parametrize('geom', GEOMS, ids=_geom_id)
def test_corr_zero_patches_vs_oracle(geom, norm, l2norm, monkeypatch):
    """A zero region in each map: all-zero Ref patches (norm 0) and all-zero query patches (every score 0, a tie
    that the lowest Ref index wins)."""
    monkeypatch.setenv('C2M_CORR_EXACT_TIES', '1')
    fin, fref = _inputs(geom, 451)
    _, C, h, w = fin.shape
    fin[0, :, 1:6, 2:8] = 0.0
    fref[0, :, 2:7, 3:10] = 0.0
    idx, val = _run(fin, fref, *norm, l2norm)
    _check(idx[0], val[0], fin[0], fref[0], *norm, l2norm)
    assert bool((val[0, 1:4, 2:6] == 0).all()) and bool((idx[0, 1:4, 2:6] == 0).all())
