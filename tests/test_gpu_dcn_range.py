"""The deformable-convolution forwards across the fp32 range and with non-finite inputs (-m gpu).

Routes:
- `ext_tc`: `_ext.dcn_v2_forward` on an eligible shape (3x3 / s1 / p1 / d1, C/dg % 8 == 0): the tensor-core kernel
  (`dcn_wgmma_kernel`, csrc/dcn_umma.cu) with the final offsets and mask as given.
- `ext_ffma`: the same call with C2M_EXT_DCN_TC=0 (`dcn_fwd_kernel`, csrc/dcn_v2.cu).
- `deform_conv_tc`: `ModulatedDeformConv` at fp32 with groups = 1, which takes the tensor-core route.
- `fused_tc`: `DCN_sep_pre_multi_offset`'s fused tail with a plain fp32 `x` and an index-map pre-offset source.
- `fused_ffma`: `dcn_v2_fused_forward` with the same inputs.

The tensor-core kernel computes with split-fp16 operands.  An fp32 input gets a per-image exponent from its largest
finite |x| (and, under the `_ext` contract, its mask one from its largest |mask|), so the result is fp32-grade at any
magnitude and scaling an image by 2^k scales its output by exactly 2^k.  A sample outside the window and a corner
outside the image are not read, as in the reference, so a NaN or Inf reaches only the outputs whose samples read it.

References: the fp64-accumulating C oracles (`c_oracle.dcn_v2_forward(acc64=True)`; `deform_conv_oracle` for
`deform_conv`, which tests/test_dcn_nonfinite_oracle.py pins against torchvision for non-finite inputs).  Each image is
checked against its own output scale.  Bars: 2e-5 on the tensor-core routes, 1e-5 on the FFMA routes at fp32, 1e-11
at fp64."""
import contextlib
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import seeding
from oracle import c_oracle
from oracle import deform_conv_oracle as dco

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32, F64 = torch.float32, torch.float64
BAR = {'ext_tc': 2e-5, 'deform_conv_tc': 2e-5, 'fused_tc': 2e-5, 'ext_ffma': 1e-5, 'fused_ffma': 1e-5}
TC_ROUTES = ['ext_tc', 'deform_conv_tc', 'fused_tc']
ROUTES = ['ext_tc', 'ext_ffma', 'deform_conv_tc', 'fused_tc', 'fused_ffma']
GEOMS = {  # (B, C, Cout, dg, H, W): the model's large layer, and Cout = 100 (L = 4, two output slices)
    'C64dg8_Cout64': (1, 64, 64, 8, 21, 19),
    'C32dg1_Cout100': (1, 32, 100, 1, 19, 13),
}
_worst = {}


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()
    yield
    if _worst:
        print('\ndcn range: largest error / bar: ' + ', '.join(f'{k} {v:.3f}' for k, v in sorted(_worst.items())))


def _is_ext(route):
    return route.startswith('ext') or route.startswith('deform_conv')


def _index_map(seed, B, H, W):
    """Scale-1 index map covering an H x W map (gh = H - 2, gw = W - 2)."""
    gh, gw = H - 2, W - 2
    return torch.from_numpy(np.random.default_rng(seed).integers(0, gh * gw, (B, gh, gw)))


def _inputs(geo, seed, x_scale=1.0):
    """x, weight, bias and both modulation sources: final (off, mask) and raw (om, idx)."""
    B, C, Cout, dg, H, W = geo
    x = seeding.randn(seed, (B, C, H, W), x_scale)
    wgt = seeding.randn(seed + 1, (Cout, C, 3, 3), 1.0 / np.sqrt(9 * C))
    bias = seeding.randn(seed + 2, (Cout,), x_scale)
    off = seeding.randn(seed + 3, (B, 18 * dg, H, W), 2.0)
    mask = torch.sigmoid(seeding.randn(seed + 4, (B, 9 * dg, H, W)))
    om = torch.cat([off, seeding.randn(seed + 5, (B, 9 * dg, H, W))], 1)
    idx = _index_map(seed + 6, B, H, W)
    return x, wgt, bias, off, mask, om, idx


def _final(om, idx, dg):
    """Final offsets and mask of the fused routes' raw inputs."""
    B = om.shape[0]
    pre = torch.stack([c_oracle.offset_pyramid(idx[b], 1) for b in range(B)]).repeat(1, dg, 1, 1, 1)
    off = om[:, :18 * dg].clone()
    off[:, 0::2] += pre[..., 1]
    off[:, 1::2] += pre[..., 0]
    return off, torch.sigmoid(om[:, 18 * dg:])


def _want(route, x, wgt, bias, off, mask, om, idx, dg, lrelu=False):
    if not _is_ext(route):
        off, mask = _final(om, idx, dg)
    out = c_oracle.dcn_v2_forward(x, wgt, bias if bias is not None else torch.zeros(wgt.shape[0]), off, mask, dg=dg,
                                  acc64=True)
    return F.leaky_relu(out, 0.1) if lrelu else out


@contextlib.contextmanager
def _env(name, value):
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        yield
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


def _got(route, x, wgt, bias, off, mask, om, idx, dg, lrelu=False):
    """Runs `route` on the GPU; CPU inputs, GPU result.  Asserts that the call took the tensor-core kernel exactly when
    the route's name says so (the tensor-core routes would otherwise fall back to FFMA unnoticed)."""
    from c2m_b200 import ops
    real, calls = ops.dcn_v2_fused_tc, []

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)
    ops.dcn_v2_fused_tc = spy
    try:
        with _env('C2M_EXT_DCN_TC', '0' if route == 'ext_ffma' else '1'), _env('C2M_DCN_TC', '1'):
            out = _run(route, x, wgt, bias, off, mask, om, idx, dg, lrelu)
    finally:
        ops.dcn_v2_fused_tc = real
    assert calls == ([1] if route.endswith('_tc') else []), (route, calls)
    return out


def _run(route, x, wgt, bias, off, mask, om, idx, dg, lrelu):
    import _ext
    from c2m_b200 import ops
    from mmsr.models.archs.DCNv2.dcn_v2 import DCN_sep_pre_multi_offset
    from mmsr.models.archs.dcn import modulated_deform_conv
    x = x if x.is_cuda else x.to(DEV)
    wgt = wgt.to(DEV)
    bias = bias.to(DEV) if bias is not None else None
    if route in ('ext_tc', 'ext_ffma'):
        b = bias if bias is not None else torch.zeros(wgt.shape[0], device=DEV)
        return _ext.dcn_v2_forward(x, wgt, b, off.to(DEV), mask.to(DEV), 3, 3, 1, 1, 1, 1, 1, 1, dg)
    if route == 'deform_conv_tc':
        return modulated_deform_conv(x, off.to(DEV), mask.to(DEV), wgt, bias, 1, 1, 1, 1, dg)
    slope = 0.1 if lrelu else 1.0
    if route == 'fused_tc':
        mod = DCN_sep_pre_multi_offset(x.shape[1], wgt.shape[0], 3, stride=1, padding=1, deformable_groups=dg).to(DEV)
        with torch.no_grad():
            mod.weight.copy_(wgt)
            if bias is None:
                mod.bias = None
            else:
                mod.bias.copy_(bias)
            return mod.fused_tail(x, om.to(DEV), types.SimpleNamespace(max_idx=idx.to(DEV), scale=1, ref_gw=None),
                                  lrelu_slope=slope)
    assert route == 'fused_ffma'
    return ops.dcn_v2_fused_forward(x, om.to(DEV), wgt, bias, dg, idx=idx.to(DEV), pre_scale=1, lrelu_slope=slope)


def _per_image_within(got, want, bar, what):
    got = got.detach().cpu().double()
    want = want.double()
    assert got.shape == want.shape, what
    for b in range(want.shape[0]):
        scale = float(want[b].abs().max())
        assert 0 < scale < float('inf'), what
        err = float((got[b] - want[b]).abs().max())
        assert err <= bar * scale, f'{what} image {b}: max abs err {err:.3e} vs scale {scale:.3e}'
        key = what.split('[')[0]
        _worst[key] = max(_worst.get(key, 0.0), err / (bar * scale))


SCALES = [1e-30, 1e-6, 1e-4, 1e-3, 1e2, 1e5, 1e30]


@pytest.mark.parametrize('scale', SCALES, ids=lambda s: f'{s:g}')
@pytest.mark.parametrize('route', ROUTES)
@pytest.mark.parametrize('geo', list(GEOMS), ids=list(GEOMS))
def test_dcn_input_scale_vs_fp64(geo, route, scale):
    """x and bias at `scale`: fp32-grade at every magnitude, like the reference's fp32 im2col + SGEMM."""
    g = GEOMS[geo]
    x, wgt, bias, off, mask, om, idx = _inputs(g, 300, scale)
    want = _want(route, x, wgt, bias, off, mask, om, idx, g[3])
    got = _got(route, x, wgt, bias, off, mask, om, idx, g[3])
    _per_image_within(got, want, BAR[route], f'scale:{route}[{scale:g}]')


@pytest.mark.parametrize('mscale', [1e-6, 1e3, 1e6], ids=lambda s: f'{s:g}')
@pytest.mark.parametrize('route', ['ext_tc', 'ext_ffma'])
@pytest.mark.parametrize('geo', list(GEOMS), ids=list(GEOMS))
def test_ext_dcn_mask_range_vs_fp64(geo, route, mscale):
    """The `_ext` mask is the final modulation and may hold any value: uniform in [-3, 3] times `mscale`, with x at
    1e2 so that |mask * x| reaches 1e8."""
    g = GEOMS[geo]
    B, C, Cout, dg, H, W = g
    x, wgt, bias, off, _, om, idx = _inputs(g, 400, 1e2)
    mask = torch.from_numpy(np.random.default_rng(401).uniform(-3, 3, (B, 9 * dg, H, W)).astype(np.float32)) * mscale
    want = _want(route, x, wgt, bias, off, mask, om, idx, dg)
    got = _got(route, x, wgt, bias, off, mask, om, idx, dg)
    _per_image_within(got, want, BAR[route], f'mask:{route}[{mscale:g}]')


@pytest.mark.parametrize('route', TC_ROUTES)
@pytest.mark.parametrize('geo', list(GEOMS), ids=list(GEOMS))
def test_dcn_tc_mixed_scale_batch(geo, route):
    """B = 3 with images at amax 1, 1e-5 and 1e5: each meets the bar against its own scale, and the batch equals its
    images run alone bit for bit."""
    _, C, Cout, dg, H, W = GEOMS[geo]
    g = (3, C, Cout, dg, H, W)
    x, wgt, _, off, mask, om, idx = _inputs(g, 500)
    amax = torch.tensor([1.0, 1e-5, 1e5])
    x = x / x.abs().amax(dim=(1, 2, 3), keepdim=True) * amax.view(3, 1, 1, 1)
    want = _want(route, x, wgt, None, off, mask, om, idx, dg)
    got = _got(route, x, wgt, None, off, mask, om, idx, dg)
    _per_image_within(got, want, BAR[route], f'mixed:{route}')
    for i in range(3):
        one = _got(route, x[i:i + 1], wgt, None, off[i:i + 1], mask[i:i + 1], om[i:i + 1], idx[i:i + 1], dg)
        assert torch.equal(got[i:i + 1], one), i


@pytest.mark.parametrize('k', [-60, -24, -11, 11, 24, 60])
@pytest.mark.parametrize('route', ROUTES)
def test_dcn_power_of_two_equivariance_bitwise(route, k):
    """out(x 2^k) == out(x) 2^k exactly (bias None; LeakyReLU on the fused routes).  Under `_ext` the mask is scaled
    by 2^j as well and the output by 2^(k + j).  Holds for any operand scale rule that is exact exponent arithmetic."""
    g = GEOMS['C64dg8_Cout64']
    x, wgt, _, off, mask, om, idx = _inputs(g, 600)
    lrelu = not _is_ext(route)
    xd = x.to(DEV)
    base = _got(route, xd, wgt, None, off, mask, om, idx, g[3], lrelu)
    for j in ([-20, 20] if route.startswith('ext') else [0]):
        got = _got(route, xd * 2.0 ** k, wgt, None, off, mask * 2.0 ** j, om, idx, g[3], lrelu)
        assert torch.equal(got, base * 2.0 ** (k + j)), (k, j, float((got - base * 2.0 ** (k + j)).abs().max()))


# ---- non-finite inputs: the finiteness pattern of the output must be the reference's
NF_GEO = (2, 16, 24, 2, 13, 11)           # B, C, Cout, dg, H, W (C/dg = 8: eligible for the tensor-core routes)
NF_CH = 5


def _places(H, W):
    return {'corner00': (0, 0), 'cornerHW': (H - 1, W - 1), 'top_mid': (0, W // 2), 'interior': (H // 2, W // 2 - 1)}


NF_ROUTES = ROUTES + ['ext_tc_channels_last', 'dc_v1_f32', 'dc_v1_f64', 'dc_mod_f64']
NF_VALUES = {'nan': float('nan'), 'pinf': float('inf'), 'ninf': float('-inf')}


def _nf_inputs(where, value, offsets, seed=700):
    """x with one non-finite element at `where` of channel NF_CH of image 0, or (where == 'offsets') finite x with
    NaN / +-Inf offsets at some taps.  offsets: 'zero' (integer sampling points: in-bounds corners of weight 0 are
    read) or 'frac' (N(0, 2))."""
    B, C, Cout, dg, H, W = NF_GEO
    x, wgt, bias, off, mask, om, idx = _inputs(NF_GEO, seed)
    if offsets == 'zero':
        off = torch.zeros_like(off)
        om[:, :18 * dg] = 0
        idx = (torch.arange(H - 2).view(-1, 1) * (W - 2) + torch.arange(W - 2)).expand(B, -1, -1).contiguous()
    if where == 'offsets':
        v = NF_VALUES[value]
        for t in (off, om):
            t[0, 3, 2, 4] = v                    # w offset of (g 0, tap 1)
            t[0, 16, H - 1, W - 1] = v           # h offset of (g 0, tap 8)
            t[1, 18 + 9, 5, 0] = v               # w offset of (g 1, tap 4)
    else:
        y0, x0 = _places(H, W)[where]
        x[0, NF_CH, y0, x0] = NF_VALUES[value]
    return x, wgt, bias, off, mask, om, idx


def _nf_run(route, x, wgt, bias, off, mask, om, idx):
    """(got, want) of one route on the non-finite inputs."""
    dg = NF_GEO[3]
    if route.startswith('dc_'):
        from mmsr.models.archs.dcn import deform_conv, modulated_deform_conv
        dt = F64 if route.endswith('f64') else F32
        xd, od, wd = x.to(DEV, dt), off.to(DEV, dt), wgt.to(DEV, dt)
        if '_v1_' in route:
            return deform_conv(xd, od, wd, 1, 1, 1, 1, dg), dco.forward(x.to(dt), wgt.to(dt), None, off.to(dt), None,
                                                                        3, 3, 1, 1, 1, 1, 1, 1, 1, dg)
        got = modulated_deform_conv(xd, od, mask.to(DEV, dt), wd, bias.to(DEV, dt), 1, 1, 1, 1, dg)
        return got, dco.forward(x.to(dt), wgt.to(dt), bias.to(dt), off.to(dt), mask.to(dt), 3, 3, 1, 1, 1, 1, 1, 1, 1, dg)
    want = _want(route.replace('_channels_last', ''), x, wgt, bias, off, mask, om, idx, dg)
    if route == 'ext_tc_channels_last':
        x = x.to(DEV).contiguous(memory_format=torch.channels_last)
        route = 'ext_tc'
    return _got(route, x, wgt, bias, off, mask, om, idx, dg), want


def _bar(route):
    return 1e-11 if route.endswith('f64') else 1e-5 if route.startswith('dc_') else \
        BAR[route.replace('_channels_last', '')]


def _same_finiteness(got, want, bar, what):
    got = got.detach().cpu().double()
    want = want.double()
    fin_g, fin_w = torch.isfinite(got), torch.isfinite(want)
    assert torch.equal(fin_g, fin_w), \
        f'{what}: {int((fin_g != fin_w).sum())} outputs differ in finiteness ({int((~fin_w).sum())} non-finite wanted)'
    for b in range(want.shape[0]):
        f = fin_w[b]
        scale = float(want[b][f].abs().max())
        err = float((got[b][f] - want[b][f]).abs().max())
        assert err <= bar * scale, f'{what} image {b}: max abs err {err:.3e} vs scale {scale:.3e}'


NF_CASES = [(w, v, o) for w in ['corner00', 'cornerHW', 'top_mid', 'interior'] for v in NF_VALUES
            for o in ('zero', 'frac')] + [('offsets', v, o) for v in NF_VALUES for o in ('zero', 'frac')]


@pytest.mark.parametrize('case', NF_CASES, ids=lambda c: '-'.join(c))
@pytest.mark.parametrize('route', NF_ROUTES)
def test_dcn_forward_nonfinite_input_matches_oracle(route, case):
    where, value, offsets = case
    got, want = _nf_run(route, *_nf_inputs(where, value, offsets))
    # a non-finite offset moves its sample out of the window: the output stays finite (tests/test_dcn_nonfinite_oracle)
    assert bool(torch.isfinite(want).all()) == (where == 'offsets')
    _same_finiteness(got, want, _bar(route), f'{route}[{"-".join(case)}]')


@pytest.mark.parametrize('det', [False, True], ids=['atomic', 'deterministic'])
@pytest.mark.parametrize('case', [c for c in NF_CASES if c[2] == 'frac' or c[0] == 'corner00'],
                         ids=lambda c: '-'.join(c))
def test_dcn_backward_nonfinite_input_matches_oracle(case, det):
    """Every gradient of `_ext.dcn_v2_backward` (fp32) and of the `deform_conv` modulated backward (fp64) has the
    oracle's finiteness pattern: the backward gathers read only the corners they must."""
    import _ext
    from mmsr.models.archs.dcn import deform_conv_cuda  # noqa: F401
    from c2m_b200 import ops
    x, wgt, bias, off, mask, _, _ = _nf_inputs(*case)
    B, C, Cout, dg, H, W = NF_GEO
    gout = seeding.randn(710, (B, Cout, H, W))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        got = _ext.dcn_v2_backward(*[t.to(DEV) for t in (x, wgt, bias, off, mask, gout)], 3, 3, 1, 1, 1, 1, 1, 1, dg)
        want = c_oracle.dcn_v2_backward(x, wgt, bias, off, mask, gout, dg=dg)
        for name, g, w in zip(('input', 'offset', 'mask', 'weight', 'bias'), got, want):
            assert torch.equal(torch.isfinite(g.cpu()), torch.isfinite(w)), f'ext grad_{name}'
        x64, w64, o64, m64, g64 = [t.double() for t in (x, wgt, off, mask, gout)]
        got = ops.deform_conv_backward(*[t.to(DEV) for t in (x64, w64, o64, m64, g64)], 3, 3, 1, 1, 1, 1, 1, 1, 1, dg)
        want = dco.backward(x64, w64, o64, m64, g64, 3, 3, 1, 1, 1, 1, 1, 1, 1, dg)
        for name, g, w in zip(('input', 'offset', 'mask', 'weight', 'bias'), got, want):
            assert torch.equal(torch.isfinite(g.cpu()), torch.isfinite(w)), f'deform_conv grad_{name}'
    finally:
        torch.use_deterministic_algorithms(prev)
