"""The tensor-core search's rescoring window, checked on the CPU (no GPU needed).

The wgmma search ranks Ref patches by (q_hi + q_lo) . r_hi, fp16 operands of x * 2^sexp with one scale exponent per
map for the whole call.  The exact rescoring only looks at candidates within `window` of the best approximate score,
so the window must cover twice the operand rounding error of any score.  This test emulates the prep's split in numpy
(float16 rounding is round-to-nearest-even with subnormals, as `__float2half_rn`) and compares the approximate scores
with the exact ones in fp64.  It leaves out the fp32 accumulation of the tensor cores, which the window covers with
its own term.  Constants mirror the CUDA sources:
- sexp: csrc/corr_aux.cu:32 (`sexp_kernel`, |x| 2^sexp <= 1024 for the map's largest |x|);
- split: csrc/corr_aux.cu:110-112 (`prep_kernel`, hi = rn(x S), lo = rn(x S - hi));
- rinv and its maximum over nonzero Ref patches: csrc/corr_aux.cu:158-159 (`rinv_kernel`);
- window: csrc/c_abi.cu:181-182 (`window_coef`, `sub_coef`) combined as in csrc/corr_aux.cu:454-456 (`rescore_kernel`).
Inputs are the dynamic-range cases of tests/test_gpu_corr_edges.py: elements far below the map's (or the batch's)
largest one land in the fp16 subnormals, where the rounding error is absolute rather than relative."""
import numpy as np
import pytest

import seeding

C = 64


def _sexp(x):
    _, e = np.frexp(np.float32(np.abs(x).max()))
    return 10 - int(e)


def _split(x, sexp):
    vs = x.astype(np.float32) * np.float32(2.0 ** sexp)
    hi = vs.astype(np.float16)
    lo = (vs - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def _patches(x):
    """[C, h, w] -> [(h-2)(w-2), 9 C] rows of 3x3 patches (any consistent K order works for dot products)."""
    v = np.lib.stride_tricks.sliding_window_view(x, (3, 3), axis=(1, 2))      # [C, gh, gw, 3, 3]
    return v.transpose(1, 2, 0, 3, 4).reshape(v.shape[1] * v.shape[2], -1)


def _windows(fin, fref, b):
    """Largest |approx - exact| per query of image b, and the new and the old window of each query (is_norm=True)."""
    si, sr = _sexp(fin), _sexp(fref)                  # one exponent per map over the whole batch
    qh, ql = _split(fin[b], si)
    rh, _ = _split(fref[b], sr)
    pq, pr = _patches(fin[b].astype(np.float64)), _patches(fref[b].astype(np.float64))
    pn = np.sqrt((_patches(fref[b].astype(np.float32)) ** 2).sum(1, dtype=np.float32))
    rinv = (np.float32(1) / (pn + np.float32(1e-5))).astype(np.float64)
    exact = (pq @ pr.T) * rinv
    approx = (_patches(qh + ql) @ _patches(rh).T) * 2.0 ** -(si + sr) * rinv
    err = np.abs(approx - exact).max(1)
    K = C * 9
    qn = np.linalg.norm(pq, axis=1)
    window_coef = 1.01 * 2.0 ** -10 + 2.0 ** -20 * ((K + 15) // 16 + 3)
    sub_coef = 1.01 * 2.0 ** -24 * np.sqrt(K)
    rinv_max = rinv[pn > 0].max()
    old = window_coef * qn
    new = old + sub_coef * (2.0 ** -si + qn * 2.0 ** -sr * rinv_max)
    return err, new, old


def _inputs(tag):
    fin = seeding.unit_features(211, C, 20, 22).numpy()
    fref = seeding.unit_features(212, C, 24, 26).numpy()
    if tag in ('q1e-7', 'q1e-8'):
        fin = (fin * np.float32(1e-7 if tag == 'q1e-7' else 1e-8)).astype(np.float32)
        fin[5, 3, 4] = 1.0
    elif tag in ('r1e-5', 'r1e-6'):
        fref = (fref * np.float32(1e-5 if tag == 'r1e-5' else 1e-6)).astype(np.float32)
        fref[7, 10, 12] = 1e3
    elif tag == 'batch1e-8':
        return np.stack([fin, fin * np.float32(1e-8)]), np.stack([fref, fref * np.float32(1e-8)])
    return fin[None], fref[None]


TAGS = ['unit', 'q1e-7', 'q1e-8', 'r1e-5', 'r1e-6', 'batch1e-8']


@pytest.mark.parametrize('tag', TAGS)
def test_rescoring_window_covers_subnormal_rounding(tag):
    """Every score's error is at most half the window (the winner and the best approximate candidate both err)."""
    fin, fref = _inputs(tag)
    for b in range(fin.shape[0]):
        err, new, _ = _windows(fin, fref, b)
        assert (err <= new / 2).all(), (b, float((err / (new / 2)).max()))


def test_window_without_subnormal_term_is_too_narrow():
    """Regression note: the window before the subnormal term (relative fp16 rounding only) misses these inputs."""
    ratio = {}
    for tag in TAGS:
        fin, fref = _inputs(tag)
        ratio[tag] = max(float((e / (o / 2)).max()) for e, _, o in (_windows(fin, fref, b) for b in range(fin.shape[0])))
    assert ratio['unit'] < 1
    assert max(ratio.values()) > 1, ratio
