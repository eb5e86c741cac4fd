"""Oracle parity AT THE BENCHMARKED SIZES (-m gpu; slow: the CPU oracle runs for tens of seconds).

BASELINE.json configs 2 and 4: the 256-channel 160x160 <-> 160x160 search, the full LR 160x160 /
Ref 500x500 forward, and the deformable convolution with REAL pyramid offsets (random index map
=> pre-offsets of up to +-157*s pixels, sampling points far outside the image, plus fractional
learned residuals) on 64ch@160^2 and on the three layers of the config-2 network.

Reference call chain restated by the oracle: mmsr/models/archs/ref_map_util.py:26-86,
DCNv2/dcn_v2.py:222-253 (+ src/cuda/dcn_v2_im2col_cuda.cu:25-54,125-195),
mmsr/models/ref_restoration_model.py:271-279."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle, ref_path
from parity_util import flips_with_gaps, full_forward_parity

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))      # physical cores for the CPU oracle
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _rel_ok(got, want, tol):
    err = float((got - want).abs().max())
    scale = float(want.abs().max())
    assert err <= tol * scale, f'max abs err {err:.3e} vs scale {scale:.3e} (tol {tol})'


# ------------------------------------------------------------------------------- config-2 search
@pytest.mark.parametrize('case', ['unit', 'zero_padded_ref'])
def test_corr_config2_vs_reference_algorithm(case):
    """One image of BASELINE config 2 at the op boundary: feature_match_index(256ch, 160x160 vs 160x160)
    on the GPU == the reference algorithm on CPU (ref_path.feature_match_index: materialised patches,
    chunked fp32 conv2d + max, strict-> merge).  Index map bit-exact; a differing query is tolerated only
    if the two candidates' fp64 scores tie to < 1e-6 (the CPU conv2d's own fp32 summation order decides
    such a query), and there may be at most 3 of them in 24 964."""
    from mmsr.models.archs.ref_map_util import feature_match_index
    fin = seeding.unit_features(101, 256, 160, 160)
    fref = seeding.unit_features(102, 256, 160, 160)
    if case == 'zero_padded_ref':
        # what the dataset's zero padding of a 500x500 Ref to 640x640 does at the relu3 grid: an all-zero
        # region (rows / cols >= 125) whose patches have norm 0 -> the 1/(0 + 1e-5) path (ref_map_util.py:63)
        fref = fref.clone()
        fref[:, 125:, :] = 0
        fref[:, :, 125:] = 0
    want_idx, want_val = ref_path.feature_match_index(fin, fref, 3, 1, 1, is_norm=True, norm_input=True)
    idx, val = feature_match_index(fin.to(DEV), fref.to(DEV), 3, 1, 1, is_norm=True, norm_input=True)
    idx, val = idx.cpu(), val.cpu()
    assert idx.dtype == torch.int64 and tuple(idx.shape) == (158, 158)
    fl = flips_with_gaps(idx, want_idx, fin, fref)
    assert len(fl) <= 3 and all(g < 1e-6 for *_, g in fl), fl[:10]
    ok = (idx == want_idx)
    np.testing.assert_allclose(val[ok].numpy(), want_val[ok].numpy(), rtol=1e-5, atol=1e-6)
    if case == 'zero_padded_ref':
        ry, rx = want_idx // 158, want_idx % 158
        assert int(((ry > 124) | (rx > 124)).sum()) == 0      # nothing matches into the zero region


# ------------------------------------------------------------------------------- config-2 full forward
def _weights():
    return (seeding.share_extractor_weights(seeding.seeded_state_dict(seeding.spec_extractor(), 11)),
            seeding.seeded_state_dict(seeding.spec_net_map(), 12), seeding.seeded_state_dict(seeding.spec_restoration_net(), 13))


def test_full_forward_config2_vs_oracle():
    """One pair of BASELINE config 2 (LR 160x160 -> 640x640, Ref 500x500 zero-padded) through the public
    pipeline vs oracle/ref_path.full_forward on the same inputs and weights.  The index map may differ from
    the oracle's only where the two candidates' fp64 scores are closer than 1e-4 (the feature maps come from
    the tensor-core convolutions here and from oneDNN there: ~1e-6 apart); given this run's own index map the SR
    image is within 1e-3 relative of the oracle restoration, and the PSNR (reference metric, against the
    bicubic input as ground-truth proxy) within 0.01 dB of the oracle's end-to-end result."""
    from c2m_b200.pipeline import RestorationPipeline, synthetic_pair
    sds = _weights()
    pipe = RestorationPipeline(DEV).load_state_dicts(*sds).place()
    img_lq, img_up, img_ref = synthetic_pair(1234, 1, 160, 500)
    r = full_forward_parity(pipe, sds, img_lq, img_up, img_ref)
    print('config-2 parity:', r)
    assert r['max_gap64_of_flips'] < 1e-4, r
    assert r['idx_flips'] <= r['queries'] // 100, r
    assert r['sr_max_rel_err'] <= 1e-3, r
    assert r['psnr_delta_db'] < 0.01, r


# ------------------------------------------------------------------------------- DCN at size
def _dcn_real_offsets(B, C, H, scale, dg, seed):
    """SURVEY §8(d) config-4 recipe: random index map -> pre-offsets by the a4/a5 rule, + N(0, 0.5^2) learned
    residuals, random mask logits; returns the raw conv_offset_mask-like tensor, the final offsets / mask the
    `_ext` boundary takes, and the index map."""
    gh = H // scale - 2
    rng = np.random.default_rng(seed)
    idx = torch.from_numpy(rng.integers(0, gh * gh, (B, gh, gh)))
    x = seeding.randn(seed + 1, (B, C, H, H))
    w = seeding.randn(seed + 2, (C, C, 3, 3), 0.05)
    b = seeding.randn(seed + 3, (C,))
    n = dg * 9
    om = torch.cat([seeding.randn(seed + 4, (B, 2 * n, H, H), 0.5), seeding.randn(seed + 5, (B, n, H, H))], 1)
    pre = torch.stack([c_oracle.offset_pyramid(idx[i], scale) for i in range(B)])       # [B,9,H,W,2] (x,y)
    off = om[:, :2 * n].clone()
    pr = pre.repeat(1, dg, 1, 1, 1)
    off[:, 0::2] += pr[..., 1]
    off[:, 1::2] += pr[..., 0]
    assert float(pre.abs().max()) > 100 * scale               # offsets really do leave the neighbourhood
    return x, w, b, om, off, torch.sigmoid(om[:, 2 * n:]), idx


@pytest.mark.parametrize('name,C,H,scale', [('config4_64ch_160', 64, 160, 1), ('cfg2_small_256ch_160', 256, 160, 1),
                                            ('cfg2_medium_128ch_320', 128, 320, 2), ('cfg2_large_64ch_640', 64, 640, 4)])
def test_dcn_real_offsets_at_size_vs_literal_oracle(name, C, H, scale):
    """Tensor-core DCN (fused prologue, pre-offsets rebuilt from idx) and the `_ext.dcn_v2_forward` boundary
    vs the literal C restatement (fp64 accumulation) at BASELINE config 4 and on the three config-2 layers
    (B=1): exercises the 32-bit index arithmetic and the out-of-image corner rules far from the identity."""
    import _ext
    from c2m_b200 import ops
    dg = 8
    x, w, b, om, off, mask, idx = _dcn_real_offsets(1, C, H, scale, dg, 900 + C + H)
    want = c_oracle.dcn_v2_forward(x, w, b, off, mask, dg=dg, acc64=True)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    got = ops.dcn_v2_fused_tc(xd, om.to(DEV), wd, bd, dg, idx=idx.to(DEV), pre_scale=scale, lrelu=False)
    _rel_ok(got.cpu(), want, 2e-5)
    got_ext = _ext.dcn_v2_forward(xd, wd, bd, off.to(DEV), mask.to(DEV), 3, 3, 1, 1, 1, 1, 1, 1, dg)
    _rel_ok(got_ext.cpu(), want, 2e-5)
