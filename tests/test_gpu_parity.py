"""GPU parity tests proper (-m gpu): the sm_90a kernels, called through the reference-shaped
boundaries (`_ext`, `feature_match_index`, the arch classes — all of which go through the C ABI),
against the golden fixtures minted from the unmodified reference and against the oracle.

Bars (BASELINE.json north_star): index maps bit-exact; floating outputs within 1e-3 relative."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import make_golden as mg
import seeding
from oracle import c_oracle, ref_path

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    # parity is stated against the reference's fp32 arithmetic: cuDNN's TF32 convolutions (torch's
    # default on Ampere+) would perturb the conv_offset_mask outputs at the 1e-3 level
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _rel_ok(got, want, tol=1e-3):
    err = float((got - want).abs().max())
    scale = float(want.abs().max())
    assert err <= tol * scale, f'max abs err {err:.3e} vs scale {scale:.3e}'


# ------------------------------------------------------------------------------- correlation
@pytest.mark.parametrize('force_generic', [False, True], ids=['wgmma', 'generic'])
@pytest.mark.parametrize('case', mg.CORR_CASES, ids=[c[0] for c in mg.CORR_CASES])
def test_feature_match_index_golden(case, force_generic, golden):
    import c2m_b200 as c2m
    from mmsr.models.archs.ref_map_util import feature_match_index
    g = golden['corr']
    name = case[0]
    fin, fref = mg.corr_inputs(case)
    for ni in (True, False):
        if force_generic:
            idx, val = c2m.corr_argmax(fin[None].to(DEV), fref[None].to(DEV), norm_input=ni, force_generic=True)
            idx, val = idx[0], val[0]
        else:
            idx, val = feature_match_index(fin.to(DEV), fref.to(DEV), 3, 1, 1, is_norm=True, norm_input=ni)
        assert idx.dtype == torch.int64 and val.dtype == torch.float32
        assert np.array_equal(idx.cpu().numpy(), g[f'{name}/ni{int(ni)}/idx'])       # bit-exact
        np.testing.assert_allclose(val.cpu().numpy(), g[f'{name}/ni{int(ni)}/val'], rtol=1e-5, atol=1e-6)


def test_corr_is_norm_false_and_strides(golden):
    import c2m_b200 as c2m
    fin, fref = mg.corr_inputs(mg.CORR_CASES[1])
    idx, val = c2m.corr_argmax(fin[None].to(DEV), fref[None].to(DEV), is_norm=False, norm_input=False)
    assert np.array_equal(idx[0].cpu().numpy(), golden['corr']['odd_c32/raw/idx'])
    np.testing.assert_allclose(val[0].cpu().numpy(), golden['corr']['odd_c32/raw/val'], rtol=1e-5, atol=1e-6)
    # strides / patch sizes other than the model's go through the generic search: check vs the C oracle
    for (p, si, sr) in ((3, 2, 1), (3, 1, 2), (2, 1, 1), (5, 2, 3)):
        fi, fr = seeding.unit_features(31, 24, 15, 17), seeding.unit_features(32, 24, 19, 16)
        want_i, want_v = c_oracle.corr_argmax(fi, fr, p, si, sr, True, True)
        idx, val = c2m.corr_argmax(fi[None].to(DEV), fr[None].to(DEV), p, si, sr, True, True)
        assert torch.equal(idx[0].cpu(), want_i), (p, si, sr)
        np.testing.assert_allclose(val[0].cpu().numpy(), want_v.numpy(), rtol=1e-5, atol=1e-6)


def test_corr_batched_and_fused_l2norm_matches_per_image_oracle():
    """B=3 in one call with the per-pixel channel normalisation fused (what
    CorrespondenceGenerationArch does) == reference semantics image by image."""
    import c2m_b200 as c2m
    f1 = seeding.randn(41, (3, 64, 36, 38))
    f2 = seeding.randn(42, (3, 64, 36, 38))
    f2[1, :, 20:, :] = 0                                    # zero-feature region (eps paths)
    idx, val = c2m.corr_argmax(f1.to(DEV), f2.to(DEV), norm_input=True, l2norm=True)
    for b in range(3):
        a = F.normalize(f1[b].reshape(64, -1), dim=0).view(64, 36, 38)
        r = F.normalize(f2[b].reshape(64, -1), dim=0).view(64, 36, 38)
        want_i, want_v, gap = c_oracle.corr_argmax(a, r, is_norm=True, norm_input=True, want_gap=True)
        bad = idx[b].cpu() != want_i
        # a mismatch is only tolerable where the fp64 margin is below fp32 resolution of the inputs
        assert int(bad.sum()) == 0 or float(gap[bad].max()) < 1e-6, (b, int(bad.sum()))
        np.testing.assert_allclose(val[b].cpu().numpy()[~bad.numpy()], want_v.numpy()[~bad.numpy()], rtol=2e-5, atol=2e-6)


def test_corr_full_size_properties():
    """BASELINE config 2 map size (256 ch, 160x160 vs 160x160) — too big for the CPU oracle in a
    test, so size-independent properties: (1) planted translation is recovered on the interior,
    (2) the tensor-core search and the generic CUDA-core search agree bit-for-bit, (3) val is the
    exact score of idx (recomputed in fp64 for a sample of queries)."""
    import c2m_b200 as c2m
    dy, dx = 5, 9
    ref = seeding.randn(51, (256, 160, 160))
    inp = torch.zeros_like(ref)
    inp[:, :160 - dy, :160 - dx] = ref[:, dy:, dx:]
    inp = inp + seeding.randn(52, (256, 160, 160), 0.05)
    nrm = lambda t: (t / t.norm(dim=0, keepdim=True).clamp_min(1e-12))
    fin, fref = nrm(inp).to(DEV), nrm(ref).to(DEV)
    idx, val = c2m.corr_argmax(fin[None], fref[None], norm_input=True)
    idx, val = idx[0].cpu(), val[0].cpu()
    yy, xx = torch.meshgrid(torch.arange(158), torch.arange(158), indexing='ij')
    want = (yy + dy) * 158 + (xx + dx)
    inner = (yy < 158 - dy) & (xx < 158 - dx)
    assert torch.equal(idx[inner], want[inner])
    idx_g, val_g = c2m.corr_argmax(fin[None], fref[None], norm_input=True, force_generic=True)
    assert torch.equal(idx_g[0].cpu(), idx) and torch.equal(val_g[0].cpu(), val)
    fi, fr = fin.double().cpu(), fref.double().cpu()
    for (qy, qx) in ((0, 0), (17, 101), (157, 157), (80, 3)):
        r = int(idx[qy, qx]); ry, rx = divmod(r, 158)
        pq, pr = fi[:, qy:qy + 3, qx:qx + 3], fr[:, ry:ry + 3, rx:rx + 3]
        s = float((pq * (pr / (pr.norm() + 1e-5))).sum() / (pq.norm() + 1e-5))
        assert abs(s - float(val[qy, qx])) < 2e-6


def test_corr_tie_flooded_input_budget_and_exact_mode(monkeypatch):
    """Smooth feature maps put most Ref patches inside every query's rescoring window.  Default: the exhaustive re-scan
    is skipped once more than max(64, queries / 256) queries overflow, and the result is the best LISTED candidate —
    within 2E (the window) of the exact maximum.  C2M_CORR_EXACT_TIES=1: always exhaustive = the oracle's argmax."""
    import c2m_b200 as c2m
    g = torch.Generator().manual_seed(21)
    def smooth(c, h, w):
        base = torch.rand(1, c, 5, 5, generator=g)
        x = F.interpolate(base, size=(h, w), mode='bicubic', align_corners=False) + 0.002 * torch.randn(1, c, h, w, generator=g)
        return x[0]
    fin, fref = smooth(64, 40, 40), smooth(64, 44, 44)
    idx_b, val_b = c2m.corr_argmax(fin[None].to(DEV), fref[None].to(DEV), norm_input=True)
    monkeypatch.setenv('C2M_CORR_EXACT_TIES', '1')
    idx_e, val_e = c2m.corr_argmax(fin[None].to(DEV), fref[None].to(DEV), norm_input=True)
    monkeypatch.delenv('C2M_CORR_EXACT_TIES')
    # exact mode against the literal fp64 oracle
    o_idx, o_val, gap = c_oracle.corr_argmax(fin, fref, is_norm=True, norm_input=True, want_gap=True)
    bad = idx_e[0].cpu() != o_idx
    assert int(bad.sum()) == 0 or float(gap[bad].max()) < 1e-6, int(bad.sum())
    # budget mode: every query's exact score is within the window of the exact maximum (val = score / (||P_q|| + 1e-5))
    K = 64 * 9
    window = 1.01 * 2.0 ** -10 + 2.0 ** -20 * (K / 16 + 3)
    short = (val_e - val_b)[0].cpu()
    assert float(short.min()) >= -1e-6 and float(short.max()) <= window * 1.01, (float(short.min()), float(short.max()))
    assert torch.isfinite(val_b).all() and int(idx_b.min()) >= 0 and int(idx_b.max()) < 42 * 42


def test_corr_error_paths():
    import c2m_b200 as c2m
    from c2m_b200._lib import C2MError
    with pytest.raises(RuntimeError, match='mismatch'):
        c2m.corr_argmax(torch.zeros(1, 8, 6, 6, device=DEV), torch.zeros(1, 16, 6, 6, device=DEV))
    with pytest.raises(C2MError, match='smaller than the patch'):
        c2m.corr_argmax(torch.zeros(1, 8, 2, 6, device=DEV), torch.zeros(1, 8, 6, 6, device=DEV))


# ------------------------------------------------------------------------------- offsets
@pytest.mark.parametrize('tag,shape', [('a', (32, 12, 12)), ('b', (16, 9, 14))])
def test_correspondence_arch_offsets_golden(tag, shape, golden):
    from mmsr.models.archs.corres_generation_arch import CorrespondenceGenerationArch
    c, h, w = shape
    net = CorrespondenceGenerationArch(3, 1, ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19')
    net.load_state_dict(seeding.seeded_state_dict(seeding.spec_net_map(), 7))
    net.to(DEV).eval()
    f1 = seeding.randn(300 + ord(tag), (2, c, h, w)).to(DEV)
    f2 = seeding.randn(400 + ord(tag), (2, c, h, w)).to(DEV)
    img_ref = seeding.rand_image(500 + ord(tag), (2, 3, 4 * h, 4 * w)).to(DEV)
    with torch.no_grad():
        pre, feats = net({'dense_features1': f1, 'dense_features2': f2}, img_ref)
    assert set(pre.keys()) == {'relu1_1', 'relu2_1', 'relu3_1'}
    for k in ('relu3_1', 'relu2_1', 'relu1_1'):
        assert np.array_equal(pre[k].cpu().numpy().astype(np.int16), golden['offsets'][f'{tag}/{k}']), k
    want_sum = float(golden['offsets'][f'{tag}/relu3_1_sum'])
    assert abs(float(feats['relu3_1'].double().sum()) - want_sum) <= 1e-3 * abs(want_sum) + 1e-2
    flow = net.index_to_flow(pre.max_idx[0])
    assert tuple(flow.shape) == (1, h, w, 2) and torch.equal(flow[0], pre['relu3_1'][0, 0])


# ------------------------------------------------------------------------------- DCN
def _dcn_case_tensors(case):
    name, b, c, cout, h, w, dg, seed, osc = case
    x = seeding.randn(seed, (b, c, h, w))
    wgt = seeding.randn(seed + 5, (cout, c, 3, 3), 0.1)
    bias = seeding.randn(seed + 6, (cout,))
    off = seeding.randn(seed + 7, (b, 2 * dg * 9, h, w), 2.0 * osc)
    off[:, :, ::2, ::3] = off[:, :, ::2, ::3].round()
    mask = torch.sigmoid(seeding.randn(seed + 8, (b, dg * 9, h, w)))
    return x, wgt, bias, off, mask


@pytest.mark.parametrize('route', ['tensor_core_when_eligible', 'ffma'])
@pytest.mark.parametrize('channels_last', [False, True])
@pytest.mark.parametrize('case', mg.DCN_CASES, ids=[c[0] for c in mg.DCN_CASES])
def test_ext_dcn_v2_forward_vs_literal_oracle(case, channels_last, route, monkeypatch):
    """B1 boundary.  3x3/s1/p1/d1 shapes with C/dg % 8 == 0 ('wide' here, every DCN of the model) are routed to
    the tensor-core kernel (split-fp16 contraction: 2e-5 of the output scale vs the fp64-accumulating oracle);
    everything else, and everything with C2M_EXT_DCN_TC=0, runs the operation-for-operation FFMA kernel (1e-5)."""
    import _ext
    from c2m_b200 import ops
    if route == 'ffma':
        monkeypatch.setenv('C2M_EXT_DCN_TC', '0')
    dg = case[6]
    x, wgt, bias, off, mask = _dcn_case_tensors(case)
    want = c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, dg=dg, acc64=True)
    xd = x.to(DEV)
    if channels_last:
        xd = xd.contiguous(memory_format=torch.channels_last)
    got = _ext.dcn_v2_forward(xd, wgt.to(DEV), bias.to(DEV), off.to(DEV), mask.to(DEV), 3, 3, 1, 1, 1, 1, 1, 1, dg)
    assert got.shape == want.shape and got.is_contiguous()
    tc = route != 'ffma' and ops.dcn_tc_supported(x.shape[1], wgt.shape[0], dg)
    _rel_ok(got.cpu(), want, 2e-5 if tc else 1e-5)


def test_ext_dcn_strided_dilated_and_big_cout():
    import _ext
    x = seeding.randn(1, (1, 8, 11, 9)); wgt = seeding.randn(2, (6, 8, 3, 3), 0.2); bias = seeding.randn(3, (6,))
    ho, wo = (11 + 4 - 5) // 2 + 1, (9 + 4 - 5) // 2 + 1
    off = seeding.randn(4, (1, 36, ho, wo), 1.5); mask = torch.sigmoid(seeding.randn(5, (1, 18, ho, wo)))
    want = c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, 3, 3, 2, 2, 2, 2, 2, 2, dg=2)
    got = _ext.dcn_v2_forward(x.to(DEV), wgt.to(DEV), bias.to(DEV), off.to(DEV), mask.to(DEV), 3, 3, 2, 2, 2, 2, 2, 2, 2)
    _rel_ok(got.cpu(), want, 1e-5)
    # Cout > 256 (several output blocks), dg = 1, 5x5 kernel (taps walked in two passes)
    x = seeding.randn(6, (1, 40, 9, 8)); wgt = seeding.randn(7, (300, 40, 5, 5), 0.05); bias = seeding.randn(8, (300,))
    off = seeding.randn(9, (1, 50, 9, 8), 2.0); mask = torch.sigmoid(seeding.randn(10, (1, 25, 9, 8)))
    want = c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, 5, 5, 1, 1, 2, 2, 1, 1, dg=1)
    got = _ext.dcn_v2_forward(x.to(DEV), wgt.to(DEV), bias.to(DEV), off.to(DEV), mask.to(DEV), 5, 5, 1, 1, 2, 2, 1, 1, 1)
    _rel_ok(got.cpu(), want, 1e-5)


def test_ext_error_behaviour():
    import _ext
    z = lambda *s: torch.zeros(*s, device=DEV)
    with pytest.raises(RuntimeError, match='kernel shape wont match'):
        _ext.dcn_v2_forward(z(1, 8, 6, 6), z(8, 8, 3, 3), z(8), z(1, 18, 6, 6), z(1, 9, 6, 6), 5, 5, 1, 1, 1, 1, 1, 1, 1)
    with pytest.raises(RuntimeError, match='kernel channels wont match'):
        _ext.dcn_v2_forward(z(1, 8, 6, 6), z(8, 4, 3, 3), z(8), z(1, 18, 6, 6), z(1, 9, 6, 6), 3, 3, 1, 1, 1, 1, 1, 1, 1)
    from c2m_b200._lib import C2MError
    with pytest.raises(C2MError, match='not divisible'):
        _ext.dcn_v2_forward(z(1, 8, 6, 6), z(8, 8, 3, 3), z(8), z(1, 54, 6, 6), z(1, 27, 6, 6), 3, 3, 1, 1, 1, 1, 1, 1, 3)


@pytest.mark.parametrize('case', mg.DCN_CASES, ids=[c[0] for c in mg.DCN_CASES])
def test_dcn_sep_pre_multi_offset_module_golden(case, golden):
    """The fused module tail == the reference module's output (golden), and the reference's own
    Python prologue on top of the drop-in `_ext` agrees too (i.e. `_ext` really is a drop-in)."""
    from mmsr.models.archs.DCNv2.dcn_v2 import DCN_sep_pre_multi_offset, dcn_v2_conv
    name, b, c, cout, h, w, dg, seed, osc = case
    m = DCN_sep_pre_multi_offset(c, cout, 3, stride=1, padding=1, dilation=1, deformable_groups=dg, extra_offset_mask=True)
    spec = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = seeding.seeded_state_dict(spec, seed + 3)
    sd['conv_offset_mask.weight'] = sd['conv_offset_mask.weight'] * osc
    m.load_state_dict(sd)
    m.to(DEV).eval()
    x, feat, pre = [t.to(DEV) for t in mg.dcn_inputs(case)]
    want = torch.from_numpy(golden['dcn'][name + '/out'])
    with torch.no_grad():
        got = m([x, feat], pre)
        _rel_ok(got.cpu(), want, 1e-4)
        # reference prologue (dcn_v2.py:229-245) in plain torch + dcn_v2_conv -> _ext
        out = m.conv_offset_mask(feat)
        o1, o2, mk = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        pr = pre.repeat([1, dg, 1, 1, 1])
        reord = torch.zeros_like(offset)
        reord[:, 0::2] = pr[..., 1]
        reord[:, 1::2] = pr[..., 0]
        got2 = dcn_v2_conv(x, offset + reord, torch.sigmoid(mk), m.weight, m.bias, 1, 1, 1, dg)
        _rel_ok(got2.cpu(), want, 1e-4)
        # fused LeakyReLU + channels-last output
        got3 = m([x, feat], pre, lrelu_slope=0.1, channels_last_out=True)
        assert got3.is_contiguous(memory_format=torch.channels_last)
        _rel_ok(got3.cpu(), F.leaky_relu(want, 0.1), 1e-4)


def test_dcn_fused_idx_equals_materialised_pre_offsets():
    import c2m_b200 as c2m
    B, C, dg, gh, gw, s = 2, 16, 4, 10, 12, 2
    H, W = s * (gh + 2), s * (gw + 2)
    idx = torch.from_numpy(np.random.default_rng(5).integers(0, gh * gw, (B, gh, gw))).to(DEV)
    x = seeding.randn(61, (B, C, H, W)).to(DEV)
    om = seeding.randn(62, (B, 27 * dg, H, W), 0.7).to(DEV)
    wgt = seeding.randn(63, (C, C, 3, 3), 0.1).to(DEV)
    bias = seeding.randn(64, (C,)).to(DEV)
    pre = c2m.offset_pyramid(idx, s)
    want_pre = torch.stack([c_oracle.offset_pyramid(idx[b].cpu(), s) for b in range(B)])
    assert torch.equal(pre.cpu(), want_pre)
    a = c2m.dcn_v2_fused_forward(x, om, wgt, bias, dg, pre_offset=pre)
    b_ = c2m.dcn_v2_fused_forward(x, om, wgt, bias, dg, idx=idx, pre_scale=s)
    assert torch.equal(a, b_)


# ------------------------------------------------------------------------------- full path
def _weights():
    return (seeding.share_extractor_weights(seeding.seeded_state_dict(seeding.spec_extractor(), 11)),
            seeding.seeded_state_dict(seeding.spec_net_map(), 12), seeding.seeded_state_dict(seeding.spec_restoration_net(), 13))


@pytest.mark.parametrize('tag', ['cfg1', 'b2'])
def test_full_forward_golden(tag, golden):
    """BASELINE config 1 (+ a B=2 variant) through extractor -> net_map -> net_g.

    Index map: bit-exact against the reference's, except that a query whose fp64 top-1/top-2 margin
    is below 1e-4 may legitimately flip, because the feature maps feeding the search come from
    cuDNN here and oneDNN in the golden run (they differ at the 1e-6 level); the search itself is
    pinned bit-exactly by the tests above.  SR: within 1e-3 relative of the oracle restoration
    evaluated on THIS run's index map (exact downstream check), and, when no index flipped,
    within 1e-3 relative / 0.01 dB PSNR of the reference's own output."""
    from c2m_b200.pipeline import RestorationPipeline
    from mmsr.utils import metrics
    from mmsr.utils.util import tensor2img
    sd_e, sd_m, sd_g = _weights()
    pipe = RestorationPipeline(DEV).load_state_dicts(sd_e, sd_m, sd_g).place()
    hr, img_lq, img_up, img_ref = seeding.full_case_inputs(tag)
    sr, idx = pipe.forward(img_lq.to(DEV), img_up.to(DEV), img_ref.to(DEV), return_idx=True)
    g = golden['full']
    want_idx = torch.from_numpy(g[tag + '/max_idx']).long()
    flipped = idx.cpu() != want_idx
    gap = torch.from_numpy(g[tag + '/gap64'])
    assert int(flipped.sum()) <= 2 and (int(flipped.sum()) == 0 or float(gap[flipped].max()) < 1e-4), \
        (int(flipped.sum()), gap[flipped])
    # downstream exactness given this run's index map
    pre = {k: torch.stack([ref_path.offset_pyramid(ref_path.index_to_flow(idx[b].cpu()))[k] for b in range(idx.shape[0])])
           for k in ('relu3_1', 'relu2_1', 'relu1_1')}
    with torch.no_grad():
        want_sr = ref_path.restoration_net(sd_g, img_lq, pre, ref_path.vgg19_ref_features(sd_m, img_ref))
    _rel_ok(sr.cpu(), want_sr, 1e-3)
    if int(flipped.sum()) == 0:
        want = torch.from_numpy(g[tag + '/sr'])
        _rel_ok(sr.cpu(), want, 1e-3)
        for i in range(sr.shape[0]):
            p_ours = metrics.psnr(tensor2img(sr[i].cpu()), tensor2img(hr[i]), crop_border=4)
            p_ref = metrics.psnr(tensor2img(want[i]), tensor2img(hr[i]), crop_border=4)
            assert abs(p_ours - p_ref) < 0.01, (p_ours, p_ref)
    # the public host->host call gives the same image
    out = pipe.run_host(img_lq.pin_memory(), img_up.pin_memory(), img_ref.pin_memory())
    assert torch.equal(out, sr.cpu())


def test_search_on_reference_features_is_bit_exact(golden):
    """Same full case, but the feature maps are computed on the HOST with the same torch ops the
    golden run used, then searched on the GPU: the index map must equal the reference's exactly."""
    import c2m_b200 as c2m
    sd_e, _, _ = _weights()
    for tag in ('cfg1', 'b2'):
        hr, img_lq, img_up, img_ref = seeding.full_case_inputs(tag)
        with torch.no_grad():
            f1, f2 = ref_path.contras_extractor(sd_e, img_up, img_ref)
        idx, _ = c2m.corr_argmax(f1.to(DEV), f2.to(DEV), norm_input=True, l2norm=True)
        want = torch.from_numpy(golden['full'][tag + '/max_idx']).long()
        bad = idx.cpu() != want
        gap = torch.from_numpy(golden['full'][tag + '/gap64'])
        # the fused in-kernel normalisation may differ from F.normalize by an ulp: only sub-1e-6 margins may flip
        assert int(bad.sum()) == 0 or float(gap[bad].max()) < 1e-6, (tag, int(bad.sum()), gap[bad])


def test_cli_runs_on_synthetic_yaml(tmp_path):
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, 'c2-matching_b200', 'mmsr', 'test.py'), '-opt',
                        os.path.join(root, 'tests', 'fixtures', 'test_c2m_synth.yml')], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert '# Validation synth # PSNR:' in r.stderr + r.stdout


def test_validation_gpu_metrics_equal_host_metrics(tmp_path):
    """N1: `validation` with device-side scores + per-pair loader workers returns the same PSNR / PSNR_Y / SSIM_Y as
    the host path (the reference's numpy / cv2 arithmetic, per-batch loader), incl. zero-padded pairs and PNG output."""
    import bench
    from mmsr.data import create_dataloader, create_dataset
    from mmsr.models.ref_restoration_model import RefRestorationModel
    opt = {'name': 'valtest', 'suffix': None, 'scale': 4, 'crop_border': None, 'dist': False, 'is_train': False,
           'network_g': {'type': 'RestorationNet', 'ngf': 64, 'n_blocks': 16, 'groups': 8},
           'network_map': {'type': 'CorrespondenceGenerationArch', 'patch_size': 3, 'stride': 1,
                           'vgg_layer_list': ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg_type': 'vgg19', 'vgg_pretrained': False},
           'network_extractor': {'type': 'ContrasExtractorSep'}, 'path': {'visualization': str(tmp_path)}}
    model = RefRestorationModel(opt)
    for net, sd in zip((model.net_extractor, model.net_map, model.net_g), bench.seeded_weights()):
        net.load_state_dict(sd, strict=True)
    dopt = {'name': 'synth', 'type': 'SyntheticRefDataset', 'phase': 'test', 'num': 5, 'gt_size': 80, 'ref_size': 96,
            'scale': 4, 'batch_size': 2, 'num_workers': 2}
    dset = create_dataset(dopt)
    a = dict(model.validation(create_dataloader(dset, dopt), 0, save_img=True, metrics_device='cuda'))
    b = dict(model.validation(create_dataloader(dset, dict(dopt, per_sample_workers=False)), 0, metrics_device='cpu'))
    c = dict(model.validation(create_dataloader(dset, dopt), 0, metrics_device='cpu'))     # host metrics behind the PairBatcher
    assert a['n'] == b['n'] == c['n'] == 5 and a['metrics_device'] == 'cuda' and b['metrics_device'] == 'cpu'
    for k in ('psnr', 'psnr_y', 'ssim_y'):
        assert abs(a[k] - b[k]) <= 1e-9 * max(1.0, abs(b[k])), (k, a[k], b[k])
        assert c[k] == b[k], (k, c[k], b[k])
    assert len(list((tmp_path / 'synth').glob('*.png'))) == 5


# ------------------------------------------------------------------------------- tensor-core 3x3 conv
@pytest.mark.parametrize('cfg', [(2, 64, 64, 40, 44, 'relu', False), (1, 64, 64, 37, 29, None, True),
                                 (1, 64, 32, 32, 32, 'lrelu', False), (1, 32, 3, 48, 40, None, False),
                                 (2, 3, 64, 32, 24, 'lrelu', False), (1, 24, 40, 33, 21, 'relu', True)],
                         ids=lambda c: f'{c[1]}to{c[2]}_{c[3]}x{c[4]}')
def test_conv3x3_psa_vs_fp64(cfg):
    """Split-fp16 tensor-core convolution: fp32-grade (<= 1e-5 of the output scale, i.e. at least as
    close to the fp64 result as cuDNN's fp32 kernels), incl. ragged tiles, padded channel counts,
    fused activation and residual."""
    from c2m_b200 import ops
    B, cin, cout, H, W, act, res = cfg
    x = seeding.randn(1, (B, cin, H, W), 1.5)
    w = seeding.randn(2, (cout, cin, 3, 3), 0.05)
    b = seeding.randn(3, (cout,), 0.5)
    r = seeding.randn(4, (B, cout, H, W)) if res else None
    want = F.conv2d(x.double(), w.double(), b.double(), 1, 1)
    want = want.relu() if act == 'relu' else F.leaky_relu(want, 0.1) if act == 'lrelu' else want
    if res:
        want = want + r.double()
    xp = ops.psa_from_f32(x.to(DEV))
    assert float((ops.psa_to_f32(xp).cpu() - x).abs().max()) <= 2e-6 * 1.5 * 5      # 22-bit split
    yp = ops.conv3x3_psa(xp, w.to(DEV), b.to(DEV), act=act, residual=ops.psa_from_f32(r.to(DEV)) if res else None)
    got = ops.psa_to_f32(yp, channels_last=True)
    assert got.is_contiguous(memory_format=torch.channels_last)
    err = float((got.cpu().double() - want).abs().max())
    assert err <= 1e-5 * float(want.abs().max()), err


def test_resblock_chain_fast_path_equals_module_path():
    from mmsr.models.archs import arch_util
    body = arch_util.make_layer(arch_util.ResidualBlockNoBN, 4, nf=64).to(DEV).eval()
    h = seeding.randn(9, (2, 64, 36, 28)).to(DEV)
    skip = seeding.randn(10, (2, 64, 36, 28)).to(DEV)
    with torch.no_grad():
        fast = arch_util.body_forward(body, h, skip=skip)
        slow = body(h) + skip
    _rel_ok(fast, slow, 2e-5)


def test_conv3x3_general_modes_vs_fp64():
    """Generalised tensor-core conv: two concatenated inputs, >64 output channels (sliced), fused
    PixelShuffle(2), fp32 strided output with an added tensor, both outputs at once."""
    from c2m_b200 import ops
    for (B, c1, c2, cout, H, W, act, mode) in ((1, 64, 256, 256, 40, 40, 'lrelu', 'psa'), (2, 64, 128, 128, 24, 40, 'lrelu', 'psa'),
                                               (1, 128, 0, 216, 36, 30, None, 'f32'), (1, 64, 0, 256, 32, 24, 'lrelu', 'ps2'),
                                               (1, 256, 0, 256, 20, 26, 'relu', 'both'), (1, 32, 0, 3, 40, 48, None, 'f32add'),
                                               (1, 64, 64, 64, 130, 70, 'lrelu', 'psa'), (1, 64, 0, 20, 24, 24, 'relu', 'f32')):
        x1 = seeding.randn(11, (B, c1, H, W), 1.2)
        x2 = seeding.randn(12, (B, c2, H, W), 0.8) if c2 else None
        w = seeding.randn(13, (cout, c1 + c2, 3, 3), 0.03)
        b = seeding.randn(14, (cout,), 0.5)
        want = F.conv2d((torch.cat([x1, x2], 1) if c2 else x1).double(), w.double(), b.double(), 1, 1)
        want = want.relu() if act == 'relu' else F.leaky_relu(want, 0.1) if act == 'lrelu' else want
        p1 = ops.psa_from_f32(x1.to(DEV))
        p2 = ops.psa_from_f32(x2.to(DEV)) if c2 else None
        wd, bd = w.to(DEV), b.to(DEV)
        if mode == 'psa':
            got = ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2))
        elif mode == 'f32':
            got = ops.conv3x3_psa(p1, wd, bd, act=act, psa_out=False, out_f32=True)
            oc = ops.conv3x3_psa(p1, wd, bd, act=act, psa_out=False, out_f32=True, f32_octets=True)
            assert oc.shape == tuple(got.shape) and torch.equal(oc.nchw(), got)
            assert float(oc.data[:, -1, :, :, cout % 8 or 8:].abs().sum()) == 0      # padding channels are zero
            cl = ops.conv3x3_psa(p1, wd, bd, act=act, psa_out=False, out_f32=True, channels_last=True)
            assert cl.is_contiguous(memory_format=torch.channels_last) and torch.equal(cl, got)
        elif mode == 'f32add':
            add = seeding.randn(15, (B, cout, H, W))
            got = ops.conv3x3_psa(p1, wd, bd, act=act, psa_out=False, out_f32=True, add_f32=add.to(DEV))
            want = want + add.double()
        elif mode == 'ps2':
            got = ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, pixel_shuffle=2))
            want = F.pixel_shuffle(want, 2)
        else:
            gp, got = ops.conv3x3_psa(p1, wd, bd, act=act, out_f32=True)
            assert float((ops.psa_to_f32(gp) - got).abs().max()) <= 1e-6 * float(want.abs().max())
        err = float((got.cpu().double() - want).abs().max())
        assert err <= 3e-5 * float(want.abs().max()), (mode, err)


def _module_path_on_idx(pipe, args, idx_given):
    """Run the pipeline's nets under the CURRENT environment switches (cuDNN convs / FFMA DCN), but feed the
    restoration net the pre-offsets of `idx_given`: isolates the conv / DCN numerics from index flips.
    Returns (sr, the index map this path would have found itself)."""
    from mmsr.models.archs.corres_generation_arch import PreOffsets
    lq, up, ref = args
    with torch.no_grad():
        feats = pipe.net_extractor(up, ref)
        pre, ref_feat = pipe.net_map(feats, ref)
        sr = pipe.net_g(lq, PreOffsets(idx_given, idx_given.shape[2]), ref_feat)
    return sr, pre.max_idx


def test_fast_conv_path_equals_cudnn_path(monkeypatch):
    """The whole pipeline with every plain conv on the tensor-core kernel vs the same pipeline with
    them on exact-fp32 cuDNN (C2M_FAST_CONV=0): same index map, SR within 1e-3 relative."""
    from c2m_b200.pipeline import RestorationPipeline
    sd_e, sd_m, sd_g = _weights()
    pipe = RestorationPipeline(DEV).load_state_dicts(sd_e, sd_m, sd_g).place()
    hr, img_lq, img_up, img_ref = seeding.full_case_inputs('b2')
    args = [t.to(DEV) for t in (img_lq, img_up, img_ref)]
    sr_fast, idx_fast = pipe.forward(*args, return_idx=True)
    monkeypatch.setenv('C2M_FAST_CONV', '0')
    sr_slow, idx_slow = _module_path_on_idx(pipe, args, idx_fast)
    assert int((idx_fast != idx_slow).sum()) <= 2
    _rel_ok(sr_fast, sr_slow, 1e-3)          # always: the module path is evaluated on the fast path's index map


@pytest.mark.parametrize('cfg', [(1, 64, 64, 8, 10, 12, 2), (2, 16, 16, 2, 20, 9, 1), (1, 128, 128, 8, 9, 9, 2),
                                 (1, 256, 256, 8, 20, 20, 1), (1, 32, 48, 4, 18, 11, 1)],
                         ids=lambda c: f'C{c[1]}to{c[2]}_dg{c[3]}')
def test_dcn_tensor_core_vs_literal_oracle(cfg):
    """tensor-core DCN (gather warps + split-fp16 contraction) == the literal C restatement of the
    reference kernel (fp64 accumulation), pre-offsets rebuilt from the index map, LeakyReLU fused,
    PSA and fp32 outputs identical."""
    import c2m_b200 as c2m
    from c2m_b200 import ops
    B, C, cout, dg, gh, gw, sc = cfg
    H, W = sc * (gh + 2), sc * (gw + 2)
    idx = torch.from_numpy(np.random.default_rng(5).integers(0, gh * gw, (B, gh, gw))).to(DEV)
    x = seeding.randn(61, (B, C, H, W)).to(DEV)
    om = seeding.randn(62, (B, 27 * dg, H, W), 0.7).to(DEV)
    wgt = seeding.randn(63, (cout, C, 3, 3), 0.1).to(DEV)
    bias = seeding.randn(64, (cout,)).to(DEV)
    gp, gf = ops.dcn_v2_fused_tc(x, om, wgt, bias, dg, idx=idx, pre_scale=sc, lrelu=True, psa_out=True, out_f32=True)
    pre = c2m.offset_pyramid(idx, sc)
    n = dg * 9
    off = om[:, :2 * n].clone()
    pr = pre.repeat(1, dg, 1, 1, 1)
    off[:, 0::2] += pr[..., 1]
    off[:, 1::2] += pr[..., 0]
    lit = c_oracle.dcn_v2_forward(x.cpu(), wgt.cpu(), bias.cpu(), off.cpu(), torch.sigmoid(om[:, 2 * n:]).cpu(), dg=dg, acc64=True)
    lit = F.leaky_relu(lit, 0.1)
    _rel_ok(gf.cpu(), lit, 2e-5)
    assert float((ops.psa_to_f32(gp) - gf).abs().max()) <= 1e-6 * float(lit.abs().max())
    # same through the pre_offset tensor instead of idx, no activation
    gf2 = ops.dcn_v2_fused_tc(x, om, wgt, bias, dg, pre_offset=pre, lrelu=False)
    ff = c2m.dcn_v2_fused_forward(x, om, wgt, bias, dg, pre_offset=pre)
    _rel_ok(gf2, ff, 2e-5)
    # offsets / mask handed over in the octet-planar fp32 layout: bit-identical result
    c8 = (27 * dg + 7) // 8
    padded = torch.zeros(B, c8 * 8, H, W, device=DEV)
    padded[:, :27 * dg] = om
    oct_om = ops.OctF32(padded.view(B, c8, 8, H, W).permute(0, 1, 3, 4, 2).contiguous(), 27 * dg)
    assert torch.equal(oct_om.nchw(), om)
    gf3 = ops.dcn_v2_fused_tc(x, oct_om, wgt, bias, dg, pre_offset=pre, lrelu=False)
    assert torch.equal(gf3, gf2)
    gf4 = ops.dcn_v2_fused_tc(x, om, wgt, bias, dg, pre_offset=pre, lrelu=False, channels_last_out=True)
    assert gf4.is_contiguous(memory_format=torch.channels_last) and torch.equal(gf4, gf2)


@pytest.mark.parametrize('cfg', [(2, 8, 6, 9, 7, 2, 3, 1, 1, 1), (1, 12, 10, 8, 10, 4, 3, 2, 2, 2), (1, 16, 16, 12, 11, 8, 3, 1, 1, 1)])
def test_ext_dcn_v2_backward_vs_oracle(cfg):
    """N4: `_ext.dcn_v2_backward` (and autograd through `dcn_v2_conv`) == the literal restatement of
    the reference backward, itself checked against torch autograd on CPU (tests/test_oracle.py)."""
    import _ext
    from mmsr.models.archs.DCNv2.dcn_v2 import dcn_v2_conv
    B, C, cout, H, W, dg, ks, st, pad, dil = cfg
    T = ks * ks
    ho, wo = (H + 2 * pad - (dil * (ks - 1) + 1)) // st + 1, (W + 2 * pad - (dil * (ks - 1) + 1)) // st + 1
    x = seeding.randn(1, (B, C, H, W)); wgt = seeding.randn(2, (cout, C, ks, ks), 0.2); bias = seeding.randn(3, (cout,))
    off = seeding.randn(4, (B, 2 * dg * T, ho, wo), 2.5)
    off = torch.where((off - off.round()).abs() < 0.05, off + 0.11, off)
    mask = torch.sigmoid(seeding.randn(5, (B, dg * T, ho, wo)))
    gout = seeding.randn(6, (B, cout, ho, wo))
    want = c_oracle.dcn_v2_backward(x, wgt, bias, off, mask, gout, ks, ks, st, st, pad, pad, dil, dil, dg)
    d = [t.to(DEV) for t in (x, wgt, bias, off, mask, gout)]
    got = _ext.dcn_v2_backward(d[0], d[1], d[2], d[3], d[4], d[5], ks, ks, st, st, pad, pad, dil, dil, dg)
    for g_, w_, name in zip(got, want, ('input', 'offset', 'mask', 'weight', 'bias')):
        assert g_.shape == w_.shape, name
        assert float((g_.cpu() - w_).abs().max()) <= 5e-5 * max(1.0, float(w_.abs().max())), name
    leaves = [t.clone().requires_grad_(True) for t in d[:5]]
    y = dcn_v2_conv(leaves[0], leaves[3], leaves[4], leaves[1], leaves[2], st, pad, dil, dg)
    y.backward(d[5])
    assert float((leaves[0].grad.cpu() - want[0]).abs().max()) <= 5e-5 * max(1.0, float(want[0].abs().max()))
    assert float((leaves[1].grad.cpu() - want[3]).abs().max()) <= 5e-5 * max(1.0, float(want[3].abs().max()))


def test_dcn_sep_pre_multi_offset_trains(golden):
    """With grad enabled the module takes the differentiable route (reference formulation over
    dcn_v2_conv -> _ext forward/backward): same output as the fused inference kernel, finite grads."""
    from mmsr.models.archs.DCNv2.dcn_v2 import DCN_sep_pre_multi_offset
    case = mg.DCN_CASES[0]
    name, b, c, cout, h, w, dg, seed, osc = case
    m = DCN_sep_pre_multi_offset(c, cout, 3, stride=1, padding=1, dilation=1, deformable_groups=dg, extra_offset_mask=True)
    sd = seeding.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed + 3)
    m.load_state_dict(sd)
    m.to(DEV)
    x, feat, pre = [t.to(DEV) for t in mg.dcn_inputs(case)]
    y = m([x, feat], pre)
    assert y.requires_grad
    _rel_ok(y.detach().cpu(), torch.from_numpy(golden['dcn'][name + '/out']), 1e-4)
    y.square().mean().backward()
    for p_ in (m.weight, m.bias, m.conv_offset_mask.weight):
        assert p_.grad is not None and torch.isfinite(p_.grad).all() and float(p_.grad.abs().sum()) > 0


def test_psa_maxpool_and_vgg_trunk_fast_path():
    from c2m_b200 import ops
    from mmsr.models.archs.vgg_arch import VGGFeatureExtractor
    x = seeding.randn(71, (2, 24, 38, 46), 2.0).to(DEV)
    got = ops.psa_to_f32(ops.psa_maxpool2(ops.psa_from_f32(x)))
    want = F.max_pool2d(x, 2, 2)
    assert float((got - want).abs().max()) <= 2e-6 * float(want.abs().max())
    net = VGGFeatureExtractor(['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19')
    net.load_state_dict(seeding.seeded_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 5))
    net.to(DEV).eval()
    img = seeding.rand_image(72, (1, 3, 96, 80)).to(DEV)
    with torch.no_grad():
        fast = net(img)
        xn = (img - net.mean) / net.std
        slow = {}
        for name, layer in net.vgg_net.named_children():
            xn = torch.relu(xn) if isinstance(layer, torch.nn.ReLU) else layer(xn)
            if name in ('relu1_1', 'relu2_1', 'relu3_1'):
                slow[name] = xn
    for k in slow:
        _rel_ok(fast[k], slow[k], 2e-5)


# ------------------------------------------------------------------------------- full-size properties
def test_dcn_full_size_reduces_to_plain_conv():
    """BASELINE config 2 large layer (64 ch, 640x640): with zero learned offsets, an identity index
    map (zero flow) and zero mask logits the deformable conv must equal 0.5 * conv3x3(x, W) + bias."""
    from c2m_b200 import ops
    C, H, dg, gh = 64, 640, 8, 158
    x = seeding.randn(81, (1, C, H, H)).to(DEV)
    w = seeding.randn(82, (C, C, 3, 3), 0.05).to(DEV)
    b = seeding.randn(83, (C,)).to(DEV)
    om = torch.zeros(1, 27 * dg, H, H, device=DEV)
    idx = torch.arange(gh * gh, device=DEV, dtype=torch.int64).view(1, gh, gh)
    got = ops.dcn_v2_fused_tc(x, om, w, b, dg, idx=idx, pre_scale=4, lrelu=False)
    want = 0.5 * F.conv2d(x, w, None, 1, 1) + b.view(1, -1, 1, 1)
    _rel_ok(got, want, 1e-4)


def test_conv_full_size_vs_cudnn_fp32():
    from c2m_b200 import ops
    x = seeding.randn(84, (1, 64, 640, 640)).to(DEV)
    w = seeding.randn(85, (64, 64, 3, 3), 0.05).to(DEV)
    b = seeding.randn(86, (64,)).to(DEV)
    got = ops.psa_to_f32(ops.conv3x3_psa(ops.psa_from_f32(x), w, b, act='relu'))
    want = F.relu(F.conv2d(x, w, b, 1, 1))
    _rel_ok(got, want, 1e-4)


def test_full_size_pipeline_is_deterministic_and_batch_invariant():
    """Config-2 shapes (LR 160, Ref 500 -> 640): two runs are bitwise identical (no atomics on the
    forward path) and image 0 of a B=2 batch equals the B=1 result (index map exactly)."""
    from c2m_b200.pipeline import RestorationPipeline, synthetic_pair
    pipe = RestorationPipeline(DEV).load_state_dicts(*_weights()).place()
    lq, up, ref = [t.to(DEV) for t in synthetic_pair(77, 2, 160, 500)]
    sr_a, idx_a = pipe.forward(lq, up, ref, return_idx=True)
    sr_b, idx_b = pipe.forward(lq, up, ref, return_idx=True)
    assert torch.equal(idx_a, idx_b) and torch.equal(sr_a, sr_b)
    sr_1, idx_1 = pipe.forward(lq[:1], up[:1], ref[:1], return_idx=True)
    assert torch.equal(idx_1[0], idx_a[0])
    _rel_ok(sr_1[0], sr_a[0], 1e-5)
    assert tuple(sr_a.shape) == (2, 3, 640, 640) and torch.isfinite(sr_a).all()


def test_cuda_graph_replay_is_bit_identical_to_eager():
    """`forward_graphed` / `run_host(cuda_graph=True)`: the forward captured once per input shape and replayed gives exactly
    the eager results, also for inputs that differ from the ones it was captured with, and for a second shape."""
    from c2m_b200.pipeline import RestorationPipeline, synthetic_pair
    pipe = RestorationPipeline(DEV, cuda_graph=True).load_state_dicts(*_weights()).place()
    first = [t.to(DEV) for t in synthetic_pair(5, 2, 40, 96)]
    pipe.forward(*first)                                    # calibration happens eagerly, before any capture
    for seed, batch, lr, rs in ((5, 2, 40, 96), (6, 2, 40, 96), (7, 1, 48, 160), (8, 2, 40, 96)):
        host = synthetic_pair(seed, batch, lr, rs)
        x = [t.to(DEV) for t in host]
        sr_e, idx_e = pipe.forward(*x, return_idx=True)
        sr_e, idx_e = sr_e.clone(), idx_e.clone()
        sr_g, idx_g = pipe.forward_graphed(*x, return_idx=True)
        assert torch.equal(idx_g, idx_e) and torch.equal(sr_g, sr_e), (seed, batch, lr)
        out = pipe.run_host(*[t.pin_memory() for t in host])
        assert torch.equal(out, sr_e.cpu())
    assert len(pipe._graphs) == 2


def test_non_square_pipeline_fast_vs_module_path(monkeypatch):
    """CUFED5-like non-square pair (LR 84x124 -> 336x496, Ref 300x420 zero-padded): tensor-core conv/DCN
    path vs the cuDNN + FFMA module path give the same index map and SR (ragged tiles on every scale)."""
    from c2m_b200.pipeline import RestorationPipeline
    pipe = RestorationPipeline(DEV).load_state_dicts(*_weights()).place()
    g = torch.Generator().manual_seed(5)
    lr_h, lr_w = 84, 124
    lq = torch.rand(1, 3, lr_h, lr_w, generator=g)
    up = F.interpolate(lq, scale_factor=4, mode='bicubic', align_corners=False).clamp(0, 1)
    ref = F.pad(torch.rand(1, 3, 300, 420, generator=g), (0, 4 * lr_w - 420, 0, 4 * lr_h - 300))
    args = [t.to(DEV) for t in (lq, up, ref)]
    sr_fast, idx_fast = pipe.forward(*args, return_idx=True)
    monkeypatch.setenv('C2M_FAST_CONV', '0')
    monkeypatch.setenv('C2M_DCN_TC', '0')
    sr_slow, idx_slow = _module_path_on_idx(pipe, args, idx_fast)
    assert tuple(sr_fast.shape) == (1, 3, 4 * lr_h, 4 * lr_w)
    assert int((idx_fast != idx_slow).sum()) <= 3
    _rel_ok(sr_fast, sr_slow, 1e-3)          # always: the module path is evaluated on the fast path's index map


# ------------------------------------------------------------------------------- PSA dynamic range
def test_psa_scale_exponent_and_range():
    """The packed-split layout stores fp16 pairs of x * 2^sa.  (1) activations spanning 1e-4 ... 1e4 with Kaiming-scale
    weights: <= 1e-5 of the output scale vs fp64, finite;  (2) a tensor that is tiny everywhere needs a scale exponent:
    with ops.suggest_sa the same bar holds (with sa = 0 its lo halves fall into the fp16 subnormals);  (3) beyond the
    fp16 range the result is non-finite and the pipeline-level check raises instead of returning garbage."""
    from c2m_b200 import ops
    rng = np.random.default_rng(7)
    w = torch.from_numpy((rng.standard_normal((64, 64, 3, 3)) * np.sqrt(2.0 / 576)).astype(np.float32))
    b = seeding.randn(3, (64,), 0.1)
    wd, bd = w.to(DEV), b.to(DEV)

    def run(x, sa_in, sa_out):
        yp = ops.conv3x3_psa(ops.psa_from_f32(x.to(DEV), sa_in), wd, bd, act='lrelu', sa_out=sa_out)
        want = F.leaky_relu(F.conv2d(x.double(), w.double(), b.double(), 1, 1), 0.1)
        got = ops.psa_to_f32(yp).cpu().double()
        return float((got - want).abs().max()) / float(want.abs().max()), bool(torch.isfinite(got).all()), float(want.abs().max())

    # (1) wide range, exponent 0
    mag = torch.from_numpy(10.0 ** rng.uniform(-4, 4, (1, 64, 40, 36))).float()
    x = mag * torch.from_numpy(rng.choice([-1.0, 1.0], (1, 64, 40, 36))).float()
    err, fin, _ = run(x, 0, 0)
    assert fin and err <= 1e-5, err
    # (2) tiny everywhere
    xs = seeding.randn(5, (1, 64, 40, 36), 1e-4)
    xs_out_scale = run(xs, 0, 0)[2]
    sa_i, sa_o = ops.suggest_sa(float(xs.abs().max())), ops.suggest_sa(xs_out_scale + 0.1 * 0 + float(b.abs().max()))
    assert sa_i >= 20
    err_s, fin_s, _ = run(xs, sa_i, sa_o)
    assert fin_s and err_s <= 1e-5, (err_s, sa_i, sa_o)
    assert abs(ops.psa_amax(ops.psa_from_f32(xs.to(DEV), sa_i)) - float(xs.abs().max())) <= 1e-3 * float(xs.abs().max())
    # (3) overflow is visible, not silent
    xb = seeding.randn(6, (1, 64, 40, 36), 3e5)
    _, fin_b, _ = run(xb, 0, 0)
    assert not fin_b
    err_b, fin_b2, _ = run(xb, ops.suggest_sa(float(xb.abs().max())), ops.suggest_sa(float(xb.abs().max()) * 3))
    assert fin_b2 and err_b <= 1e-5, err_b


def test_vgg_trunk_calibrates_nonzero_scale_exponents():
    """run_trunk calibrates a PSA scale exponent per internal activation on its first call (tapped outputs stay at 0) and
    the result still matches the plain modules; invalidate_packs drops the calibration."""
    from c2m_b200 import ops
    from mmsr.models.archs.vgg_arch import VGGFeatureExtractor
    net = VGGFeatureExtractor(['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19', pretrained=False)
    net.load_state_dict(seeding.seeded_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 5))
    net.to(DEV).eval()
    img = seeding.rand_image(72, (1, 3, 96, 80)).to(DEV)
    with torch.no_grad():
        fast = net(img)
        sa = dict(net.vgg_net._c2m_sa)
        assert any(v != 0 for k, v in sa.items()) and 'relu1_1' not in sa and 'relu2_1' not in sa, sa
        fast2 = net(img)                               # second call: cached exponents, identical result
        xn = (img - net.mean) / net.std
        slow = {}
        for name, layer in net.vgg_net.named_children():
            xn = torch.relu(xn) if isinstance(layer, torch.nn.ReLU) else layer(xn)
            if name in ('relu1_1', 'relu2_1', 'relu3_1'):
                slow[name] = xn
    for k in slow:
        _rel_ok(fast[k], slow[k], 2e-5)
        assert torch.equal(fast[k], fast2[k])
    ops.invalidate_packs(net)
    assert not hasattr(net.vgg_net, '_c2m_sa')
