"""Deformable PS-ROI pooling kernels behind `_ext` (csrc/psroi.cu, -m gpu) against the plain-C oracle
(oracle/psroi_oracle.c), fp32 and fp64, with and without translations.

A CTA of `psroi_fwd_kernel` / `psroi_bwd_kernel` owns one ROI's run of bins (all P*P bins unless P*P*S*S exceeds the
2048-entry sample table: `S7` cases with P = 7 take two runs) and one class's run of channels (8..64; few ROIs split the
channels into several runs).  Case ids name P, part_size, S, the class count K, the scale and the trans_std.

Kernel and oracle evaluate every sample position with the same correctly rounded operations in the same order (the
kernel forbids FMA contraction there), so counts must match bit for bit even for non-dyadic scales.  The boundary cases
(ROIs crossing every border, `.5` and inverted corners) still use dyadic ROIs, scales and translations so that every
position is exact in fp32.

Bars: counts bit-exact; output 1e-5 (fp32) / 1e-12 (fp64) of the output scale; each gradient 1e-5 / 1e-10 of its own
largest magnitude; grad_trans identical bit for bit over two runs.  Each check prints its error as a fraction of its
bar."""
import pytest
import torch

from oracle import psroi_oracle

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BARS = {torch.float32: (1e-5, 1e-5), torch.float64: (1e-12, 1e-10)}


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


def _frac(got, want, bar, what):
    want = want.double()
    err = float((got.detach().cpu().double() - want).abs().max()) if want.numel() else 0.0
    scale = float(want.abs().max()) if want.numel() else 0.0
    assert err <= bar * max(scale, 1e-300), f'{what}: max abs err {err:.3e} vs scale {scale:.3e}'
    f = err / (bar * scale) if scale > 0 else 0.0
    print(f'[psroi bar] {what}: {f:.3g} of bar')
    return f


def _make(seed, B, C, H, W, R, K, part, scale, dtype, dyadic=True, bad_batch=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    span_w, span_h = W / scale, H / scale
    lo = torch.tensor([-0.25 * span_w, -0.25 * span_h])
    hi = torch.tensor([1.2 * span_w, 1.2 * span_h])
    c = torch.rand(R, 4, generator=g, dtype=torch.float64) * (hi - lo).repeat(2) + lo.repeat(2)
    c = torch.floor(c * 2) / 2                          # half-integers: exercises round-half-away-from-zero
    c[::5, 2:] = c[::5, :2] - 3                         # inverted ROIs
    c[1::7, 2:] = c[1::7, :2]                           # zero-size ROIs
    b = torch.randint(0, B, (R, 1), generator=g).double()
    if bad_batch:
        b[::3] = torch.tensor([-1.0, float(B), B + 0.5, -0.5])[torch.arange(len(b[::3])) % 4][:, None]
    trans = torch.randn(R, 2 * K, part, part, generator=g, dtype=torch.float64)
    if dyadic:
        trans = torch.floor(trans * 64) / 64
    return x.to(dtype), torch.cat([b, c], 1).to(dtype), trans.to(dtype)


# id: (B, C, H, W, R, K, P, part, S, scale, trans_std)
CASES = {
    'P1_part1_S1_K1_s1by4_t0.1': (2, 8, 12, 15, 9, 1, 1, 1, 1, 0.25, 0.1),
    'P3_part5_S2_K3_s1by2_t0.1': (2, 24, 16, 13, 11, 3, 3, 5, 2, 0.5, 0.1),
    'P7_part7_S4_K1_s1by16_t0.1': (2, 16, 20, 24, 13, 1, 7, 7, 4, 1 / 16, 0.1),
    'P7_part3_S7_K3_s1by3_t0': (2, 12, 14, 17, 7, 3, 7, 3, 7, 1 / 3, 0.0),
    'P3_part2_S4_K1_s1by3_t0.1': (1, 8, 9, 9, 10, 1, 3, 2, 4, 1 / 3, 0.1),
    'P7_part7_S2_K3_s1by4_t0': (2, 9, 10, 12, 6, 3, 7, 7, 2, 0.25, 0.0),
    'readme_B2_C32_64x64_R20_P7_S4': (2, 32, 64, 64, 20, 1, 7, 7, 4, 0.25, 0.1),
    'slices_C203_R3_P7_S4': (1, 203, 12, 12, 3, 1, 7, 7, 4, 0.5, 0.1),
    'R0': (1, 8, 8, 8, 0, 1, 3, 3, 2, 0.5, 0.1),
}


def _run(case, dtype, no_trans, seed=0, bad_batch=False):
    B, C, H, W, R, K, P, part, S, scale, tstd = CASES[case]
    x, bbox, trans = _make(seed, B, C, H, W, R, K, part, scale, dtype, dyadic=True, bad_batch=bad_batch)
    args = (no_trans, scale, C, 1, P, part, S, tstd)
    return x, bbox, trans, args


def _check_case(x, bbox, trans, args, dtype, what):
    import _ext
    fbar, gbar = BARS[dtype]
    xd, bd, td = x.to(DEV), bbox.to(DEV), trans.to(DEV)
    out, cnt = _ext.dcn_v2_psroi_pooling_forward(xd, bd, td, *args)
    want_o, want_c = psroi_oracle.forward(x, bbox, trans, *args)
    assert out.dtype == dtype and cnt.dtype == dtype and out.shape == want_o.shape
    assert torch.equal(cnt.cpu(), want_c), f'{what}: counts differ'
    if want_o.numel():
        _frac(out, want_o, fbar, f'{what} output')
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64).to(dtype)
    gi, gt = _ext.dcn_v2_psroi_pooling_backward(gout.to(DEV), xd, bd, td, cnt, *args)
    wgi, wgt = psroi_oracle.backward(gout, x, bbox, trans, want_c, *args)
    assert gi.shape == x.shape and gt.shape == trans.shape and gi.dtype == dtype and gt.dtype == dtype
    if wgi.abs().max() > 0:
        _frac(gi, wgi, gbar, f'{what} grad_input')
    else:
        assert torch.equal(gi.cpu(), torch.zeros_like(wgi))
    if args[0]:
        assert torch.equal(gt.cpu(), torch.zeros_like(trans))
    elif wgt.numel() and wgt.abs().max() > 0:
        _frac(gt, wgt, gbar, f'{what} grad_trans')
        _, gt2 = _ext.dcn_v2_psroi_pooling_backward(gout.to(DEV), xd, bd, td, cnt, *args)
        assert torch.equal(gt, gt2), f'{what}: grad_trans differs between two runs'
    else:
        assert torch.equal(gt.cpu(), torch.zeros_like(wgt))


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
@pytest.mark.parametrize('no_trans', [0, 1])
@pytest.mark.parametrize('case', list(CASES))
def test_psroi_vs_oracle(case, no_trans, dtype):
    x, bbox, trans, args = _run(case, dtype, no_trans)
    _check_case(x, bbox, trans, args, dtype, f'{case} no_trans={no_trans} {dtype}')


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['f32', 'f64'])
def test_psroi_invalid_batch_index_pools_to_zero(dtype):
    """Batch indices -1, B, B + 0.5 (-> B) are outside [0, B): output 0, count 0, no gradient; -0.5 truncates to 0."""
    x, bbox, trans, args = _run('P3_part5_S2_K3_s1by2_t0.1', dtype, 0, seed=4, bad_batch=True)
    import _ext
    out, cnt = _ext.dcn_v2_psroi_pooling_forward(x.to(DEV), bbox.to(DEV), trans.to(DEV), *args)
    bi = bbox[:, 0].double().trunc()
    bad = (bi < 0) | (bi >= x.shape[0])
    assert bad.any() and (~bad).any()
    assert torch.equal(cnt[bad.to(DEV)], torch.zeros_like(cnt[bad.to(DEV)]))
    _check_case(x, bbox, trans, args, dtype, f'bad batch {dtype}')


def test_psroi_boundary_rois_exact_counts():
    """Dyadic ROIs crossing every border of a 16x16 map at scale 1/2, exact in fp32: both dtypes count the same."""
    rois = []
    for (x1, y1, x2, y2) in [(-9, 4, 7, 20), (20, 4, 40, 20), (4, -9, 20, 7), (4, 20, 20, 40), (-9, -9, 40, 40),
                             (30, 30, 31, 31), (-0.5, -0.5, 30.5, 30.5), (0.5, 1.5, 2.5, 3.5), (10, 10, 6, 6)]:
        rois.append([0, x1, y1, x2, y2])
    bbox = torch.tensor(rois, dtype=torch.float64)
    x = torch.randn(1, 6, 16, 16, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    trans = torch.floor(torch.randn(len(rois), 4, 3, 3, dtype=torch.float64) * 16) / 16
    for no_trans in (0, 1):
        args = (no_trans, 0.5, 6, 1, 3, 3, 4, 0.25)
        counts = []
        for dtype in (torch.float32, torch.float64):
            _check_case(x.to(dtype), bbox.to(dtype), trans.to(dtype), args, dtype, f'boundary no_trans={no_trans}')
            counts.append(psroi_oracle.forward(x.to(dtype), bbox.to(dtype), trans.to(dtype), *args)[1].double())
        assert torch.equal(counts[0], counts[1])
        assert (counts[1] == 0).any() and (counts[1] == 16).any() and ((counts[1] > 0) & (counts[1] < 16)).any()


def test_psroi_rejects_bad_arguments_on_gpu():
    import _ext
    x = torch.randn(1, 4, 8, 8, device=DEV)
    bbox = torch.tensor([[0, 1, 1, 5, 5]], dtype=torch.float32, device=DEV)
    trans = torch.zeros(1, 4, 3, 3, device=DEV)
    ok = (0, 0.5, 4, 1, 3, 3, 2, 0.1)
    out, cnt = _ext.dcn_v2_psroi_pooling_forward(x, bbox, trans, *ok)
    for args, t, msg in [((0, 0.5, 3, 1, 3, 3, 2, 0.1), trans, 'input channels and output channels must equal'),
                         ((0, 0.5, 4, 2, 3, 3, 2, 0.1), trans, 'group_size must be 1'),
                         ((0, 0.5, 4, 1, 0, 3, 2, 0.1), trans, 'must be >= 1'),
                         ((0, 0.5, 4, 1, 3, 0, 2, 0.1), trans, 'must be >= 1'),
                         ((0, 0.5, 4, 1, 3, 3, 0, 0.1), trans, 'must be >= 1'),
                         (ok, torch.zeros(1, 4, 2, 3, device=DEV), r'trans must be \[R, 2K, part_size, part_size\]'),
                         (ok, torch.zeros(2, 4, 3, 3, device=DEV), r'trans must be \[R, 2K'),
                         (ok, torch.zeros(1, 3, 3, 3, device=DEV), r'trans must be \[R, 2K'),
                         (ok, torch.zeros(1, 6, 3, 3, device=DEV), 'multiple of the number of trans classes'),
                         (ok, trans.double(), 'must be torch.float32'),
                         (ok, trans.cpu(), 'must be a CUDA tensor')]:
        with pytest.raises(RuntimeError, match=msg):
            _ext.dcn_v2_psroi_pooling_forward(x, bbox, t, *args)
        if args[2] == 4 and args[4] >= 1:
            with pytest.raises(RuntimeError, match=msg):
                _ext.dcn_v2_psroi_pooling_backward(torch.ones_like(out), x, bbox, t, cnt, *args)
    with pytest.raises(RuntimeError, match='must be a CUDA tensor'):
        _ext.dcn_v2_psroi_pooling_forward(x, bbox.cpu(), trans, *ok)
    # no_trans: trans may be anything, grad_trans is zeros_like(trans)
    out2, cnt2 = _ext.dcn_v2_psroi_pooling_forward(x, bbox, x.new(), 1, 0.5, 4, 1, 3, 3, 2, 0.1)
    gi, gt = _ext.dcn_v2_psroi_pooling_backward(torch.ones_like(out2), x, bbox, x.new(), cnt2, 1, 0.5, 4, 1, 3, 3, 2, 0.1)
    assert gt.shape == (0,) and gi.shape == x.shape
    # empty input map: zero gradients
    xe = torch.randn(1, 4, 0, 8, device=DEV)
    oe, ce = _ext.dcn_v2_psroi_pooling_forward(xe, bbox, trans, *ok)
    assert torch.equal(ce, torch.zeros_like(ce)) and torch.equal(oe, torch.zeros_like(oe))
    gi, gt = _ext.dcn_v2_psroi_pooling_backward(torch.ones_like(oe), xe, bbox, trans, ce, *ok)
    assert gi.shape == xe.shape and torch.equal(gt, torch.zeros_like(trans))


def test_psroi_gradcheck_fp64():
    """torch.autograd.gradcheck through dcn_v2_pooling.  The ROIs keep every sample inside (0, W-1) x (0, H-1), at
    least 1e-5 from an integer (a perturbation of 1e-6 in trans moves a sample by under 1e-6), so finite differences
    never cross a skip, a clamp or a floor.  grad_input is summed
    with atomics in no fixed order, so repeated backward passes may differ in the last bits: hence nondet_tol."""
    from mmsr.models.archs.DCNv2.dcn_v2 import dcn_v2_pooling
    from test_psroi_oracle import restate
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 4, 12, 12, generator=g, dtype=torch.float64)
    bbox = torch.tensor([[0, 3, 2, 8, 9], [1, 2, 4, 9, 7], [1, 4, 3, 6, 8]], dtype=torch.float64)
    trans = torch.randn(3, 4, 2, 2, generator=g, dtype=torch.float64) * 0.3
    args = (1.0, 3, 4, False, 1, 2, 3, 0.1)          # spatial_scale, pooled, output_dim, no_trans, group, part, S, std
    _, _, pr = restate(x, bbox, trans, 0, 1.0, 4, 3, 2, 3, 0.1, parts=True)
    w, h = pr['w'], pr['h']
    assert pr['keep'].all() and (w > 0).all() and (w < 11).all() and (h > 0).all() and (h < 11).all()
    assert ((w - w.round()).abs() > 1e-5).all() and ((h - h.round()).abs() > 1e-5).all()
    xd = x.to(DEV).requires_grad_()
    td = trans.to(DEV).requires_grad_()
    bd = bbox.to(DEV)
    assert torch.autograd.gradcheck(lambda a, t: dcn_v2_pooling(a, bd, t, *args), (xd, td), eps=1e-6, atol=1e-7,
                                    nondet_tol=1e-12)


class _OraclePooling(torch.autograd.Function):
    """dcn_v2_pooling on the CPU oracle (same argument list)."""

    @staticmethod
    def forward(ctx, input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1,
                part_size=None, sample_per_part=4, trans_std=.0):
        ctx.args = (int(no_trans), spatial_scale, output_dim, group_size, pooled_size,
                    pooled_size if part_size is None else part_size, sample_per_part, trans_std)
        out, cnt = psroi_oracle.forward(input, rois, offset, *ctx.args)
        ctx.save_for_backward(input, rois, offset, cnt)
        return out

    @staticmethod
    def backward(ctx, gout):
        input, rois, offset, cnt = ctx.saved_tensors
        gi, gt = psroi_oracle.backward(gout, input, rois, offset, cnt, *ctx.args)
        return gi, None, gt, None, None, None, None, None, None, None, None


@pytest.mark.parametrize('no_trans', [False, True])
def test_dcn_pooling_modules_vs_oracle_composition(no_trans, monkeypatch):
    """DCNPooling (last fc layer randomised) and DCNv2Pooling on the GPU against the same modules with the pooling
    swapped for the oracle, fp64: output, grad of the input, of the given translations and of every fc parameter."""
    from mmsr.models.archs.DCNv2 import dcn_v2 as mod
    torch.manual_seed(0)
    x, bbox, _ = _make(3, 2, 16, 20, 24, 12, 1, 7, 0.25, torch.float64)
    m = mod.DCNPooling(0.25, 7, 16, no_trans, trans_std=0.1, deform_fc_dim=64).double()
    if not no_trans:
        with torch.no_grad():
            m.offset_mask_fc[4].weight.normal_(0, 0.2)
            m.offset_mask_fc[4].bias.normal_(0, 0.2)
    offs = torch.randn(12, 2, 5, 5, dtype=torch.float64) * 0.5
    m2 = mod.DCNv2Pooling(0.25, 7, 16, no_trans, part_size=5, sample_per_part=3, trans_std=0.1)
    gen = torch.Generator().manual_seed(1)
    gout = torch.randn(12, 16, 7, 7, generator=gen, dtype=torch.float64)

    def run(dev, pool):
        monkeypatch.setattr(mod, 'dcn_v2_pooling', pool)
        mm = m.to(dev)
        mm.zero_grad()
        xi = x.to(dev).requires_grad_()
        oi = offs.to(dev).requires_grad_()
        y = mm(xi, bbox.to(dev))
        y2 = m2(xi, bbox.to(dev), oi)
        ((y * gout.to(dev)).sum() + (y2 * gout.to(dev)).sum()).backward()
        grads = {k: p.grad.detach().cpu().clone() for k, p in mm.named_parameters()}
        return y.detach().cpu(), y2.detach().cpu(), xi.grad.cpu(), None if no_trans else oi.grad.cpu(), grads
    got = run(DEV, mod._DCNv2Pooling.apply)
    want = run('cpu', _OraclePooling.apply)
    fbar, gbar = BARS[torch.float64]
    _frac(got[0], want[0], fbar, f'DCNPooling no_trans={no_trans} output')
    _frac(got[1], want[1], fbar, f'DCNv2Pooling no_trans={no_trans} output')
    _frac(got[2], want[2], gbar, f'modules no_trans={no_trans} grad_input')
    if not no_trans:
        _frac(got[3], want[3], gbar, 'DCNv2Pooling grad_offset')
    assert set(got[4]) == set(want[4])
    for k in got[4]:
        if want[4][k].abs().max() > 0:
            _frac(got[4][k], want[4][k], gbar, f'DCNPooling grad {k}')


def test_readme_example_through_ext_and_dcn_pooling_without_sync():
    """The reference DCNv2 README's pooling example (DCNv2/README.md:19-40), forward and backward, through `_ext` and
    DCNPooling, with any host synchronisation an error."""
    import _ext
    from mmsr.models.archs.DCNv2.dcn_v2 import DCNPooling
    torch.manual_seed(0)
    input = torch.randn(2, 32, 64, 64).cuda()
    batch_inds = torch.randint(2, (20, 1)).cuda().float()
    x = torch.randint(256, (20, 1)).cuda().float()
    y = torch.randint(256, (20, 1)).cuda().float()
    w = torch.randint(64, (20, 1)).cuda().float()
    h = torch.randint(64, (20, 1)).cuda().float()
    rois = torch.cat((batch_inds, x, y, x + w, y + h), dim=1)
    dpooling = DCNPooling(spatial_scale=1.0 / 4, pooled_size=7, output_dim=32, no_trans=False, group_size=1,
                          trans_std=0.1).cuda()
    input.requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        dout = dpooling(input, rois)
        dout.sum().backward()
        o, c = _ext.dcn_v2_psroi_pooling_forward(input.detach(), rois, input.new(), 1, 0.25, 32, 1, 7, 7, 4, 0.1)
        gi, gt = _ext.dcn_v2_psroi_pooling_backward(torch.ones_like(o), input.detach(), rois, input.new(), c, 1, 0.25,
                                                    32, 1, 7, 7, 4, 0.1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert dout.shape == (20, 32, 7, 7) and input.grad.shape == input.shape
    assert torch.isfinite(dout).all() and torch.isfinite(input.grad).all()
    want_o, want_c = psroi_oracle.forward(input.detach().cpu(), rois.cpu(), None, 1, 0.25, 32, 1, 7, 7, 4, 0.1)
    assert torch.equal(c.cpu(), want_c)
    _frac(o, want_o, 1e-5, 'README example output')
    # zero-initialised last fc layer: no translation, modulation sigmoid(0) = 1/2
    _frac(dout, 0.5 * want_o, 1e-5, 'README example DCNPooling output')
