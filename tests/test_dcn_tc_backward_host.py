"""CPU-side checks of the tensor-core DCN backward: argument checks and messages of its C entry points, their ctypes
bindings, and invalidate_packs dropping the dgrad weight pack."""
import ctypes

import pytest
import torch


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from c2m_b200 import _lib
    return _lib.lib()


def _args(**kw):
    from c2m_b200 import _lib
    a = _lib.DcnTcGradArgs()
    p = 64
    a.gy_hi = a.gy_lo = a.gy_amax = a.x_il = a.x_amax = a.mask_amax = a.offset = a.mask = p
    a.packed_w = a.grad_offset = a.grad_mask = a.grad_weight = a.ws = p
    a.B, a.C, a.H, a.W, a.Cout, a.dg = 1, 64, 16, 8, 64, 8
    a.ws_bytes = 1 << 20
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize('entry', ['c2m_dcn_tc_dgrad', 'c2m_dcn_tc_wgrad'])
def test_entry_points_validate_arguments(lib, entry):
    fn = getattr(lib, entry)
    assert fn(None, None) == 1 and b'null arguments' in lib.c2m_last_error()
    for field in ('gy_hi', 'x_il', 'offset', 'mask_amax'):
        assert fn(ctypes.addressof(_args(**{field: None})), None) == 1
        assert b'null pointer' in lib.c2m_last_error()
    assert fn(ctypes.addressof(_args(B=0)), None) == 1 and b'bad shape' in lib.c2m_last_error()
    assert fn(ctypes.addressof(_args(C=60)), None) == 1 and b'unsupported' in lib.c2m_last_error()
    assert fn(ctypes.addressof(_args(Cout=257)), None) == 1 and b'unsupported' in lib.c2m_last_error()
    assert fn(ctypes.addressof(_args(H=15)), None) == 1 and b'smaller than one pixel tile' in lib.c2m_last_error()
    assert fn(ctypes.addressof(_args(x_il=64 + 16)), None) == 1 and b'32 B aligned' in lib.c2m_last_error()
    field = 'grad_mask' if entry == 'c2m_dcn_tc_dgrad' else 'grad_weight'
    assert fn(ctypes.addressof(_args(**{field: None})), None) == 1 and b'null pointer' in lib.c2m_last_error()


def test_pack_and_sizes(lib):
    p = ctypes.c_void_p(64)
    assert lib.c2m_dcn_tc_pack_dgrad_weights_f32(None, 64, 64, 8, p, None) == 1
    assert b'null pointer' in lib.c2m_last_error()
    assert lib.c2m_dcn_tc_pack_dgrad_weights_f32(p, 60, 64, 8, p, None) == 1
    assert b'unsupported' in lib.c2m_last_error()
    assert lib.c2m_dcn_tc_dgrad_packed_weight_bytes(60, 64, 8) == 0
    # 64 channels, dg 8: 576 columns in 9 chunks of 64, 64 output channels in 2 K pieces of 4 octets, hi and lo
    assert lib.c2m_dcn_tc_dgrad_packed_weight_bytes(64, 64, 8) == 256 + 9 * 2 * 2 * 4 * 64 * 16
    # 32 channels, dg 1: 288 columns in 4 chunks of 64 and a last chunk with 32 real columns, one K piece
    assert lib.c2m_dcn_tc_dgrad_packed_weight_bytes(32, 32, 1) == 256 + 5 * 1 * 2 * 4 * 64 * 16
    assert lib.c2m_dcn_tc_wgrad_workspace_bytes(1, 60, 16, 8, 64, 8) == 0
    assert b'bad shape' in lib.c2m_last_error()


def test_symbols_are_bound():
    from c2m_b200 import _lib
    assert {'c2m_dcn_tc_dgrad_packed_weight_bytes', 'c2m_dcn_tc_pack_dgrad_weights_f32', 'c2m_dcn_tc_dgrad',
            'c2m_dcn_tc_wgrad_workspace_bytes', 'c2m_dcn_tc_wgrad'} <= set(_lib.SYMBOLS)


def test_invalidate_packs_drops_the_dcn_dgrad_pack():
    from c2m_b200 import ops
    w = torch.zeros(64, 64, 3, 3)
    w.__dict__['_c2m_dcn_pack_dgrad'] = ('tag', None, None, None)
    ops.invalidate_packs(w)
    assert '_c2m_dcn_pack_dgrad' not in w.__dict__


def test_dcn_v2_tc_rejects_cpu_tensors():
    from c2m_b200 import ops
    x, off, m, w = torch.zeros(1, 64, 16, 8), torch.zeros(1, 144, 16, 8), torch.zeros(1, 72, 16, 8), torch.zeros(64, 64, 3, 3)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.dcn_v2_tc(x, off, m, w, None, 8)
