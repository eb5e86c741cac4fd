"""The tensor-core search's rescoring window, checked on the CPU (no GPU needed).

The wgmma search ranks Ref patches by (q_hi + q_lo) . r_hi, fp16 operands of x * 2^sexp with one scale exponent per
map and image, taken from the image's largest finite |x|.  Scores are formed in search units (the score times
2^sexp_in for normalised scores), with the Ref column scale rinv = 1 / (||P_r|| 2^sexp_ref + 1e-5 2^sexp_ref), so
no product of scales leaves fp32's range.  The exact rescoring only looks at candidates within `window` of the best
approximate score, so the window must cover twice the operand rounding error of any score.  This test emulates the
prep's split in numpy (float16 rounding is round-to-nearest-even with subnormals, as `__float2half_rn`) and compares
the approximate scores with the exact ones in fp64.  It leaves out the fp32 accumulation of the tensor cores, which
the window covers with its own term.  Constants mirror the CUDA sources:
- sexp: csrc/corr_aux.cu (`sexp_kernel`, |x| 2^sexp <= 1024 for the image's largest finite |x|, clamped to +-126);
- split: csrc/corr_aux.cu (`prep_kernel`, hi = rn(x S), lo = rn(x S - hi));
- rinv and its maximum over nonzero Ref patches: csrc/corr_aux.cu (`rinv_kernel`);
- window: csrc/c_abi.cu (`window_coef`, `sub_coef`) combined as in csrc/corr_aux.cu (`rescore_kernel`).
Inputs are the dynamic-range cases of tests/test_gpu_corr_edges.py, where elements far below the map's largest one
land in the fp16 subnormals (the rounding error is absolute rather than relative), and maps far from unit scale: a
batch whose second image is the first times 1e-20, and a query map at 1e30 against a Ref map at 1e-30."""
import numpy as np
import pytest

import seeding

C = 64


def _sexp(x):
    """Exponent of one image's map: from its largest finite |x|."""
    a = np.abs(x)
    _, e = np.frexp(np.float32(a[np.isfinite(a)].max()))
    return min(126, max(-126, 10 - int(e)))


def _split(x, sexp):
    vs = x.astype(np.float32) * np.float32(2.0 ** sexp)
    hi = vs.astype(np.float16)
    lo = (vs - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def _patches(x):
    """[C, h, w] -> [(h-2)(w-2), 9 C] rows of 3x3 patches (any consistent K order works for dot products)."""
    v = np.lib.stride_tricks.sliding_window_view(x, (3, 3), axis=(1, 2))      # [C, gh, gw, 3, 3]
    return v.transpose(1, 2, 0, 3, 4).reshape(v.shape[1] * v.shape[2], -1)


def _windows(fin, fref, b, per_image=True, p_one=False):
    """Largest |approx - exact| per query of image b, the window of each query with and without its subnormal term,
    and the spread (largest - smallest exact score) of each query (is_norm=True), all in search units.
    per_image=False: one exponent per map for the whole batch (the rule before per-image exponents); p_one=True: the
    Ref factor P of the window taken as its bound 1 instead of the image's largest ||P_r|| rinv_r."""
    si, sr = (_sexp(fin[b]), _sexp(fref[b])) if per_image else (_sexp(fin), _sexp(fref))
    qh, ql = _split(fin[b], si)
    rh, _ = _split(fref[b], sr)
    pq, pr = _patches(fin[b].astype(np.float64)), _patches(fref[b].astype(np.float64))
    pn = np.sqrt((_patches(fref[b].astype(np.float32)) ** 2).sum(1, dtype=np.float32))
    exact = (pq @ pr.T) / (pn.astype(np.float64) + 1e-5) * 2.0 ** si
    # the kernels' column scale: from the scaled square sums, 1 / (||P_r|| 2^sr + 1e-5 2^sr) in fp32
    rs = (fref[b].astype(np.float32) * np.float32(2.0 ** sr)).astype(np.float32)
    pns = np.sqrt((_patches(rs) ** 2).sum(1, dtype=np.float32))
    rinv = (np.float32(1) / (pns + np.float32(1e-5 * 2.0 ** sr))).astype(np.float64)
    approx = (_patches(qh + ql) @ _patches(rh).T) * rinv
    err = np.abs(approx - exact).max(1)
    K = C * 9
    qn = np.linalg.norm(pq, axis=1) * 2.0 ** si
    window_coef = 1.01 * 2.0 ** -10 + 2.0 ** -20 * ((K + 15) // 16 + 3)
    sub_coef = 1.01 * 2.0 ** -24 * np.sqrt(K)
    rinv_max = rinv[pns > 0].max()
    P = 1.0 if p_one else float((pns.astype(np.float64) * rinv).max())
    old = window_coef * qn * P
    new = old + sub_coef * (P + qn * rinv_max)
    return err, new, old, exact.max(1) - exact.min(1)


def _inputs(tag):
    fin = seeding.unit_features(211, C, 20, 22).numpy()
    fref = seeding.unit_features(212, C, 24, 26).numpy()
    if tag in ('q1e-7', 'q1e-8'):
        fin = (fin * np.float32(1e-7 if tag == 'q1e-7' else 1e-8)).astype(np.float32)
        fin[5, 3, 4] = 1.0
    elif tag in ('r1e-5', 'r1e-6'):
        fref = (fref * np.float32(1e-5 if tag == 'r1e-5' else 1e-6)).astype(np.float32)
        fref[7, 10, 12] = 1e3
    elif tag in ('batch1e-8', 'batch1e-20'):
        s = np.float32(1e-8 if tag == 'batch1e-8' else 1e-20)
        return np.stack([fin, fin * s]), np.stack([fref, fref * s])
    elif tag == 'q1e30_r1e-30':
        fin, fref = fin * np.float32(1e30), fref * np.float32(1e-30)
    elif tag == 'r1e-20':
        fref = fref * np.float32(1e-20)
    return fin[None], fref[None]


TAGS = ['unit', 'q1e-7', 'q1e-8', 'r1e-5', 'r1e-6', 'batch1e-8', 'batch1e-20', 'q1e30_r1e-30', 'r1e-20']
# maps without elements far below their image's largest one: the window is a small fraction of the score spread
SCALED = ['unit', 'batch1e-20', 'q1e30_r1e-30', 'r1e-20']


@pytest.mark.parametrize('tag', TAGS)
def test_rescoring_window_covers_subnormal_rounding(tag):
    """Every score's error is at most half the window (the winner and the best approximate candidate both err)."""
    fin, fref = _inputs(tag)
    for b in range(fin.shape[0]):
        err, new, _, _ = _windows(fin, fref, b)
        assert (err <= new / 2).all(), (b, float((err / (new / 2)).max()))


@pytest.mark.parametrize('tag', SCALED)
def test_rescoring_window_is_small_against_the_score_spread(tag):
    """The window follows the image's score scale: below 1 % of every query's score spread, whatever the map scales
    (a Ref map at 1e-20 puts every normalised score ~1e-14 below ||P_q||, the + 1e-5 dominating its norm)."""
    fin, fref = _inputs(tag)
    for b in range(fin.shape[0]):
        _, new, _, spread = _windows(fin, fref, b)
        assert (new < 1e-2 * spread).all(), (b, float((new / spread).max()))


def test_window_with_ref_factor_one_floods_a_small_ref_map():
    """Regression note: bounding ||P_r|| rinv_r by 1 under is_norm makes the window of a Ref map at 1e-20 larger than
    every query's whole score spread: every candidate is inside it and every query overflows."""
    fin, fref = _inputs('r1e-20')
    _, new, _, spread = _windows(fin, fref, 0, p_one=True)
    assert (new > spread).all(), float((new / spread).min())


def test_window_without_subnormal_term_is_too_narrow():
    """Regression note: the window before the subnormal term (relative fp16 rounding only) misses these inputs, and
    with one exponent per map for the whole batch, the dim image of batch1e-8 too."""
    ratio = {}
    for tag in ['unit', 'q1e-7', 'q1e-8', 'r1e-5', 'r1e-6']:
        fin, fref = _inputs(tag)
        ratio[tag] = float((lambda e, n, o, s: (e / (o / 2)).max())(*_windows(fin, fref, 0)))
    assert ratio['unit'] < 1
    assert max(ratio.values()) > 1, ratio
    fin, fref = _inputs('batch1e-8')
    err, _, old, _ = _windows(fin, fref, 1, per_image=False)
    assert float((err / (old / 2)).max()) > 1

