"""Ordered `grad_input` (-m gpu): the c2m_*_det entry points against the ordered oracle (oracle/ordered_grad_oracle.c,
pinned on the CPU by tests/test_deterministic_oracle.py), bit for bit, and the backward entries of `c2m_b200.ops` with
torch's deterministic algorithms on.

Each entry point is called on a given gcol (DCN) or out_grad / top_count (PS-ROI) inside sentinel guards, so a write
outside grad_input or an element left unwritten fails the test.  The result must not change with a workspace that
holds one plane per pass, nor between calls."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from oracle import deform_conv_oracle as dco
from oracle import ordered_grad_oracle as ogo
from oracle import psroi_oracle
from test_gpu_deform_conv import CASES, _case_id, _inputs, _out_hw
from test_gpu_psroi import CASES as PS_CASES
from test_gpu_psroi import _make

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32, F64 = torch.float32, torch.float64
SFX = {F32: 'f32', F64: 'f64'}
BWD_BAR = {F32: 1e-5, F64: 1e-10}
SENTINEL = 1.5e30
GUARD = 4096


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


def _guarded(shape, dtype):
    buf = torch.full((GUARD + torch.Size(shape).numel() + GUARD,), SENTINEL, dtype=dtype, device=DEV)
    return buf, buf[GUARD:GUARD + torch.Size(shape).numel()].view(shape)


def _check_guarded(buf, inner, what):
    assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all()), f'{what}: wrote outside'
    assert not bool((inner == SENTINEL).any()), f'{what}: left elements unwritten'


def _ws(query, s, planes):
    from c2m_b200 import _lib
    n = query(s, planes)
    assert n > 0, _lib.lib().c2m_last_error().decode()
    return torch.empty(n, dtype=torch.uint8, device=DEV)


def _run_entry(fn, args_before, shape_struct, out_shape, dtype, ws):
    from c2m_b200 import _lib
    buf, gx = _guarded(out_shape, dtype)
    rc = fn(*args_before, shape_struct, gx.data_ptr(), ws.data_ptr(), ws.numel(),
            torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'det entry')
    torch.cuda.synchronize()
    _check_guarded(buf, gx, 'grad_input')
    return gx.clone()


# ---------------------------------------------------------------------------------------------------------------- DCN
def _dcn_shape(x_shape, geo, dg, dtype):
    from c2m_b200 import ops
    x = torch.empty(x_shape, dtype=dtype, device='meta')
    Ho, Wo = _out_hw(geo, *x_shape[2:])
    out = torch.empty(x_shape[0], 1, Ho, Wo, device='meta')
    return ops._shape(x, 1, *geo, dg, out)


def _dcn_det_all(gcol, off, mask, x_shape, geo, dg, dtype, entry):
    """Runs `entry` with the workspace the ops layer would give it and with a one-plane workspace, twice; returns the
    result after checking that all runs agree bit for bit."""
    from c2m_b200 import _lib
    L = _lib.lib()
    s = _dcn_shape(x_shape, geo, dg, dtype)
    fn = getattr(L, entry)
    args = (gcol.data_ptr(), off.data_ptr(), None if mask is None else mask.data_ptr())
    nplanes = x_shape[0] * dg
    res = []
    for planes in (nplanes, 1, nplanes):
        res.append(_run_entry(fn, args, s, x_shape, dtype, _ws(L.c2m_dcn_col2im_det_workspace_bytes, s, planes)))
    assert torch.equal(res[0], res[1]), 'one plane per pass changed the result'
    assert torch.equal(res[0], res[2]), 'a repeated call changed the result'
    return res[0]


def _gcol(case, seed, modulated, dtype):
    geo, B, C, Cout, groups, dg, H, W = case
    x, wgt, bias, off, mask, gout = _inputs(case, seed, modulated, dtype)
    T = geo[0] * geo[1]
    wg = wgt.double().reshape(groups, Cout // groups, -1)
    gg = gout.double().reshape(B, groups, Cout // groups, -1)
    gcol = torch.matmul(wg.transpose(1, 2), gg).reshape(B, C * T, -1).to(dtype)
    return x, gcol, off, mask


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('modulated', [False, True], ids=['v1', 'modulated'])
@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_deform_conv_col2im_det_equals_ordered_oracle(case, modulated, dtype):
    geo, B, C, Cout, groups, dg, H, W = case
    x, gcol, off, mask = _gcol(case, 500 + 10 * CASES.index(case), modulated, dtype)
    want = ogo.deform_col2im(gcol, off, mask, x.shape, *geo, dg)
    gd, od, md = [t.to(DEV) if t is not None else None for t in (gcol, off, mask)]
    got = _dcn_det_all(gd, od, md, tuple(x.shape), geo, dg, dtype, f'c2m_deform_conv_col2im_det_{SFX[dtype]}')
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize('case', [CASES[i] for i in (0, 1, 2, 5)], ids=_case_id)
def test_ext_call_of_col2im_det_equals_ordered_oracle(case):
    """c2m_deform_conv_col2im_det_f32 as `_ext.dcn_v2_backward` calls it: fp32 with a mask."""
    geo, B, C, Cout, groups, dg, H, W = case
    x, gcol, off, mask = _gcol(case, 600 + 10 * CASES.index(case), True, F32)
    want = ogo.deform_col2im(gcol, off, mask, x.shape, *geo, dg)
    got = _dcn_det_all(gcol.to(DEV), off.to(DEV), mask.to(DEV), tuple(x.shape), geo, dg, F32,
                       'c2m_deform_conv_col2im_det_f32')
    assert torch.equal(got.cpu(), want)


def _abs_offsets(B, dg, geo, H, W, h_at, w_at):
    """Offsets that move every sampling point to (h_at, w_at)."""
    kh, kw, sh, sw, ph, pw, dh, dw = geo
    Ho, Wo = _out_hw(geo, H, W)
    k = torch.arange(kh * kw)
    base_h = (torch.arange(Ho) * sh - ph)[None, :, None] + ((k // kw) * dh)[:, None, None]
    base_w = (torch.arange(Wo) * sw - pw)[None, None, :] + ((k % kw) * dw)[:, None, None]
    off = torch.stack([h_at - base_h.expand(-1, Ho, Wo), w_at - base_w.expand(-1, Ho, Wo)], 1).double()
    return off.reshape(1, 1, 2 * kh * kw, Ho, Wo).expand(B, dg, -1, -1, -1).reshape(B, 2 * dg * kh * kw, Ho, Wo)


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('where', ['one_point', 'one_pixel_map', 'outside'])
def test_deform_conv_col2im_det_extreme_maps(where, dtype):
    """one_point: every sampling point at (3.25, 5.5), so four pixels get segments of T*P entries each and all other
    segments are empty; one_pixel_map: a 1x1 input whose only pixel gets every point's in-image corner (one segment
    of T*P entries); outside: every point outside the window, every segment empty and the result exactly +0."""
    geo, B, C, dg = (3, 3, 1, 1, 1, 1, 1, 1), 2, 8, 2
    H, W = (1, 1) if where == 'one_pixel_map' else (12, 14)
    h_at, w_at = {'one_point': (3.25, 5.5), 'one_pixel_map': (0.0, 0.0), 'outside': (-7.0, 100.5)}[where]
    off = _abs_offsets(B, dg, geo, H, W, h_at, w_at).to(dtype)
    Ho, Wo = _out_hw(geo, H, W)
    gcol = torch.randn(B, C * 9, Ho * Wo, generator=torch.Generator().manual_seed(4), dtype=F64).to(dtype)
    mask = torch.rand(B, dg * 9, Ho, Wo, generator=torch.Generator().manual_seed(5), dtype=F64).to(dtype)
    want = ogo.deform_col2im(gcol, off, mask, (B, C, H, W), *geo, dg)
    got = _dcn_det_all(gcol.to(DEV), off.to(DEV), mask.to(DEV), (B, C, H, W), geo, dg, dtype,
                       f'c2m_deform_conv_col2im_det_{SFX[dtype]}').cpu()
    assert torch.equal(got, want)
    if where == 'outside':
        assert torch.equal(got, torch.zeros_like(got)) and not bool(torch.signbit(got).any())
    else:
        assert int((got != 0).sum()) > 0


def test_det_workspace_query_does_not_grow_with_batch():
    from c2m_b200 import _lib
    L = _lib.lib()
    geo = (3, 3, 1, 1, 1, 1, 1, 1)
    one = {B: L.c2m_dcn_col2im_det_workspace_bytes(_dcn_shape((B, 16, 20, 24), geo, 4, F32), 1) for B in (1, 8)}
    assert one[1] > 0 and one[1] == one[8]
    assert L.c2m_dcn_col2im_det_workspace_bytes(_dcn_shape((8, 16, 20, 24), geo, 4, F32), 32) > one[8]
    ps = {}
    for B in (1, 8):
        s = _lib.PsroiShape(B=B, C=8, H=12, W=15, R=9, no_trans=1, num_classes=1, spatial_scale=0.25, trans_std=0.1,
                            output_dim=8, group_size=1, pooled_size=3, part_size=3, sample_per_part=2)
        ps[B] = L.c2m_psroi_grad_input_det_workspace_bytes(s, 1)
    assert ps[1] > 0 and ps[1] == ps[8]


def test_det_rejects_planes_beyond_32bit_ids_and_small_workspace():
    from c2m_b200 import _lib
    L = _lib.lib()
    s = _dcn_shape((1, 1, 40000, 40000), (3, 3, 1, 1, 1, 1, 1, 1), 1, F32)    # 4 * 9 * 1.6e9 entries
    assert L.c2m_dcn_col2im_det_workspace_bytes(s, 1) == 0
    assert b'32-bit' in L.c2m_last_error()
    s = _dcn_shape((1, 4, 8, 8), (3, 3, 1, 1, 1, 1, 1, 1), 1, F32)
    ws = torch.empty(64, dtype=torch.uint8, device=DEV)
    x = torch.zeros(1, 4, 8, 8, device=DEV)
    rc = L.c2m_deform_conv_col2im_det_f32(x.data_ptr(), x.data_ptr(), None, s, x.data_ptr(), ws.data_ptr(), 64,
                                          torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b'workspace' in L.c2m_last_error()


# ------------------------------------------------------------------------------------------------------------- PS-ROI
def _psroi_det_all(gout, bbox, trans, cnt, x_shape, args, dtype):
    from c2m_b200 import _lib, ops
    L = _lib.lib()
    s = _lib.PsroiShape(B=x_shape[0], C=x_shape[1], H=x_shape[2], W=x_shape[3], R=bbox.shape[0],
                        no_trans=int(bool(args[0])), num_classes=1 if args[0] else trans.shape[1] // 2,
                        spatial_scale=args[1], trans_std=args[7], output_dim=args[2], group_size=args[3],
                        pooled_size=args[4], part_size=args[5], sample_per_part=args[6])
    fn = getattr(L, f'c2m_psroi_pooling_grad_input_det_{SFX[dtype]}')
    ptrs = (gout.data_ptr(), bbox.data_ptr(), None if args[0] else trans.data_ptr(), cnt.data_ptr())
    nplanes = x_shape[0] * s.num_classes
    res = []
    for planes in (nplanes, 1, nplanes):
        ws = _ws(L.c2m_psroi_grad_input_det_workspace_bytes, s, planes) if s.R else \
            torch.empty(0, dtype=torch.uint8, device=DEV)
        res.append(_run_entry(fn, ptrs, s, x_shape, dtype, ws))
    assert torch.equal(res[0], res[1]), 'one plane per pass changed the result'
    assert torch.equal(res[0], res[2]), 'a repeated call changed the result'
    del ops
    return res[0]


@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
@pytest.mark.parametrize('bad_batch', [False, True], ids=['', 'bad_batch'])
@pytest.mark.parametrize('no_trans', [0, 1])
@pytest.mark.parametrize('case', list(PS_CASES))
def test_psroi_grad_input_det_equals_ordered_oracle(case, no_trans, bad_batch, dtype):
    B, C, H, W, R, K, P, part, S, scale, tstd = PS_CASES[case]
    x, bbox, trans = _make(7, B, C, H, W, R, K, part, scale, dtype, dyadic=True, bad_batch=bad_batch)
    args = (no_trans, scale, C, 1, P, part, S, tstd)
    _, cnt = psroi_oracle.forward(x, bbox, trans, *args)
    cnt = cnt.clone()
    cnt.view(-1)[::5] = 0
    gout = torch.randn(cnt.shape, generator=torch.Generator().manual_seed(9), dtype=F64).to(dtype)
    want = ogo.psroi_grad_input(gout, x.shape, bbox, trans, cnt, *args)
    got = _psroi_det_all(gout.to(DEV), bbox.to(DEV), trans.to(DEV), cnt.to(DEV), tuple(x.shape), args, dtype)
    assert torch.equal(got.cpu(), want)
    if R == 0:
        assert not bool(torch.signbit(got).any()) and not bool(got.any())


# ----------------------------------------------------------------------------------------------- autograd with the flag
class _Spy:
    """Records which library entry points the ops layer calls."""

    def __init__(self, monkeypatch, names):
        from c2m_b200 import _lib
        L = _lib.lib()
        self.calls = []
        for n in names:
            f = getattr(L, n)

            def wrap(*a, _f=f, _n=n):
                self.calls.append(_n)
                return _f(*a)
            monkeypatch.setattr(L, n, wrap)


_DCN_ENTRIES = ['c2m_deform_conv_col2im_f32', 'c2m_deform_conv_col2im_f64', 'c2m_deform_conv_col2im_det_f32',
                'c2m_deform_conv_col2im_det_f64',
                'c2m_psroi_pooling_backward_f32', 'c2m_psroi_pooling_backward_f64',
                'c2m_psroi_pooling_grad_input_det_f32', 'c2m_psroi_pooling_grad_input_det_f64']


@pytest.fixture
def deterministic(request, monkeypatch):
    monkeypatch.setenv('CUBLAS_WORKSPACE_CONFIG', ':4096:8')
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param[0], warn_only=request.param[1])
    yield request.param[0]
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


FLAG = [(True, False), (True, True), (False, False)]
FLAG_IDS = ['det', 'det_warn_only', 'atomic']


def _dcn_modules(kind, dtype):
    from mmsr.models.archs.dcn import DeformConv, ModulatedDeformConv
    from mmsr.models.archs.DCNv2.dcn_v2 import DCNv2
    torch.manual_seed(0)
    if kind == 'DCNv2':
        return DCNv2(8, 12, 3, stride=1, padding=1, deformable_groups=2).to(DEV)
    if kind == 'DeformConv':
        return DeformConv(8, 12, 3, stride=1, padding=1, groups=2, deformable_groups=2).to(DEV, dtype)
    return ModulatedDeformConv(8, 12, 3, stride=1, padding=1, groups=2, deformable_groups=4).to(DEV, dtype)


@pytest.mark.parametrize('deterministic', FLAG, ids=FLAG_IDS, indirect=True)
@pytest.mark.parametrize('kind,dtype', [('DCNv2', F32), ('DeformConv', F32), ('DeformConv', F64),
                                        ('ModulatedDeformConv', F32), ('ModulatedDeformConv', F64)],
                         ids=['DCNv2', 'DeformConv-f32', 'DeformConv-f64', 'ModulatedDeformConv-f32',
                              'ModulatedDeformConv-f64'])
def test_dcn_modules_take_the_selected_col2im_path(kind, dtype, deterministic, monkeypatch):
    m = _dcn_modules(kind, dtype)
    dg = m.deformable_groups
    B, H, W = 2, 9, 11
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 8, H, W, generator=g, dtype=F64).to(dtype)
    off = (torch.floor(torch.randn(B, 18 * dg, H, W, generator=g, dtype=F64) * 128) / 64).to(dtype)
    mask = torch.rand(B, 9 * dg, H, W, generator=g, dtype=F64).to(dtype) if kind != 'DeformConv' else None
    gout = torch.randn(B, 12, H, W, generator=g, dtype=F64).to(dtype)
    spy = _Spy(monkeypatch, _DCN_ENTRIES)
    xd = x.to(DEV).requires_grad_(True)
    y = m(xd, off.to(DEV)) if mask is None else m(xd, off.to(DEV), mask.to(DEV))
    y.backward(gout.to(DEV))
    det_calls = [c for c in spy.calls if '_det_' in c]
    atomic_calls = [c for c in spy.calls if '_det_' not in c]
    if deterministic:
        assert det_calls and not atomic_calls, spy.calls
    else:
        assert atomic_calls and not det_calls, spy.calls
    groups = getattr(m, 'groups', 1)
    w = m.weight.detach().cpu()
    want = dco.backward(x, w.to(dtype), off, mask, gout, 3, 3, 1, 1, 1, 1, 1, 1, groups, dg)[0]
    err = float((xd.grad.cpu().double() - want.double()).abs().max())
    assert err <= BWD_BAR[dtype] * float(want.abs().max())


@pytest.mark.parametrize('deterministic', FLAG, ids=FLAG_IDS, indirect=True)
@pytest.mark.parametrize('no_trans', [False, True])
@pytest.mark.parametrize('dtype', [F32, F64], ids=['f32', 'f64'])
def test_dcnv2_pooling_takes_the_selected_grad_input_path(no_trans, dtype, deterministic, monkeypatch):
    from mmsr.models.archs.DCNv2.dcn_v2 import DCNv2Pooling
    x, bbox, _ = _make(3, 2, 16, 20, 24, 12, 1, 7, 0.25, dtype)
    offs = (torch.randn(12, 2, 5, 5, generator=torch.Generator().manual_seed(2), dtype=F64) * 0.5).to(dtype)
    m = DCNv2Pooling(0.25, 7, 16, no_trans, part_size=5, sample_per_part=3, trans_std=0.1)
    gout = torch.randn(12, 16, 7, 7, generator=torch.Generator().manual_seed(1), dtype=F64).to(dtype)
    spy = _Spy(monkeypatch, _DCN_ENTRIES)
    xd = x.to(DEV).requires_grad_(True)
    y = m(xd, bbox.to(DEV), offs.to(DEV))
    y.backward(gout.to(DEV))
    det = [c for c in spy.calls if '_det_' in c]
    if deterministic:
        assert det, spy.calls
    else:
        assert not det and spy.calls, spy.calls
    args = (no_trans, 0.25, 16, 1, 7, 5, 3, 0.1)
    _, cnt = psroi_oracle.forward(x, bbox, offs, *args)
    want = psroi_oracle.backward(gout, x, bbox, offs, cnt, *args)[0]
    err = float((xd.grad.cpu().double() - want.double()).abs().max())
    assert err <= BWD_BAR[dtype] * float(want.abs().max())


_SUBPROCESS = r'''
import sys, torch
sys.path[:0] = sys.argv[1:]
torch.use_deterministic_algorithms(True)
from mmsr.models.archs.dcn import DeformConv, ModulatedDeformConv
from mmsr.models.archs.DCNv2.dcn_v2 import DCNv2, DCNPooling
dev = 'cuda:0'


def grads(make, inputs):
    out = []
    for _ in range(2):
        torch.manual_seed(0)
        m = make().to(dev)
        leaves = [t.clone().requires_grad_(True) for t in inputs]
        y = m(*leaves)
        y.backward(torch.ones_like(y) * torch.linspace(-1, 1, y.numel(), device=dev).view_as(y))
        out.append([t.grad.clone() for t in leaves if t.grad is not None] +
                   [p.grad.clone() for p in m.parameters() if p.grad is not None])
    return out


g = torch.Generator(device=dev).manual_seed(1)
x = torch.randn(2, 16, 24, 28, device=dev, generator=g)
off = torch.randn(2, 18 * 4, 24, 28, device=dev, generator=g) * 2
mask = torch.rand(2, 9 * 4, 24, 28, device=dev, generator=g)
rois = torch.tensor([[0, 4., 4., 60., 50.], [1, 10., 0., 90., 80.], [0, 0., 20., 40., 90.]], device=dev)
cases = {
    'DCNv2': (lambda: DCNv2(16, 16, 3, 1, 1, deformable_groups=4), [x, off, mask]),
    'DeformConv': (lambda: DeformConv(16, 16, 3, padding=1, groups=2, deformable_groups=4), [x, off]),
    'ModulatedDeformConv': (lambda: ModulatedDeformConv(16, 16, 3, padding=1, groups=2, deformable_groups=4),
                            [x, off, mask]),
    'DCNPooling': (lambda: DCNPooling(0.25, 7, 16, False, trans_std=0.1, deform_fc_dim=64), [x]),
}
for name, (make, inputs) in cases.items():
    if name == 'DCNPooling':
        a, b = grads(lambda: _Pool(make()), inputs)
    else:
        a, b = grads(make, inputs)
    assert len(a) == len(b) and a, name
    for u, v in zip(a, b):
        assert torch.equal(u, v), name
    print(name, 'identical', len(a), 'gradients')
'''


_POOL = r'''
class _Pool(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m
        with torch.no_grad():
            m.offset_mask_fc[4].weight.normal_(0, 0.2)
            m.offset_mask_fc[4].bias.normal_(0, 0.2)

    def forward(self, x):
        return self.m(x, rois)
'''


def test_two_runs_bitwise_identical_in_a_deterministic_process():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = _SUBPROCESS.replace("cases = {", _POOL + "\ncases = {")
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=':4096:8', C2M_VGG_PRETRAINED='0')
    r = subprocess.run([sys.executable, '-c', code, root, os.path.join(root, 'c2-matching_b200')],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert 'Warning' not in r.stderr or 'deterministic' not in r.stderr, r.stderr
    for name in ('DCNv2', 'DeformConv', 'ModulatedDeformConv', 'DCNPooling'):
        assert f'{name} identical' in r.stdout, r.stdout
