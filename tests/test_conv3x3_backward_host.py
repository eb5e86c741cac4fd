"""CPU-side checks of the differentiable tensor-core 3x3 convolution: argument checks of ops.conv3x3 and of the backward's
C entry points, the dgrad weight pack dropped by invalidate_packs, and the routing module staying nn.Conv2d off the GPU."""
import ctypes

import pytest
import torch
import torch.nn.functional as F


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from c2m_b200 import _lib
    return _lib.lib()


def test_conv3x3_rejects_cpu_and_wrong_dtype():
    from c2m_b200 import ops
    x, w = torch.zeros(1, 8, 18, 10), torch.zeros(4, 8, 3, 3)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.conv3x3(x, w)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.conv3x3(x.double(), w.double())
    with pytest.raises(TypeError):
        ops.conv3x3(x.numpy(), w)


def test_wgrad_entry_points_validate_arguments(lib):
    from c2m_b200 import _lib
    p = ctypes.c_void_p(16)
    assert lib.c2m_conv3x3_wgrad(None, p, p, p, p, 1, 8, 8, 18, 10, p, p, 1 << 20, None) == 1
    assert b'null pointer' in lib.c2m_last_error()
    assert lib.c2m_conv3x3_wgrad(p, p, p, p, p, 0, 8, 8, 18, 10, p, p, 1 << 20, None) == 1
    assert lib.c2m_conv3x3_wgrad(p, p, p, p, p, 1, 8, 8, 17, 10, p, p, 1 << 20, None) == 1
    assert b'smaller than one halo tile' in lib.c2m_last_error()
    assert lib.c2m_conv3x3_wgrad_workspace_bytes(1, 0, 8, 18, 10) == 0
    assert b'bad shape' in lib.c2m_last_error()
    assert set(('c2m_conv3x3_wgrad', 'c2m_conv3x3_wgrad_workspace_bytes')) <= set(_lib.SYMBOLS)
    assert not {'c2m_grad_psa_from_f32', 'c2m_grad_unscale_f32'} & set(_lib.SYMBOLS)


def test_per_image_entry_points_validate_arguments(lib):
    """c2m_conv3x3_operand_f32 and c2m_conv3x3_wgrad_scaled reject null pointers and empty shapes with status 1 and a
    message, and per-image input exponents are refused for a concatenated input."""
    from c2m_b200 import _lib
    p = ctypes.c_void_p(16)
    for args in ((None, 1, 8, 18, 10, 0, 0, 0, 0, p, p, p), (p, 1, 8, 18, 10, 0, 0, 0, 0, None, p, p),
                 (p, 1, 8, 18, 10, 0, 0, 0, 0, p, None, p), (p, 1, 8, 18, 10, 0, 0, 0, 0, p, p, None),
                 (p, 0, 8, 18, 10, 0, 0, 0, 0, p, p, p), (p, 1, 0, 18, 10, 0, 0, 0, 0, p, p, p),
                 (p, 1, 8, 0, 10, 0, 0, 0, 0, p, p, p), (p, 1, 8, 18, 0, 0, 0, 0, 0, p, p, p)):
        assert lib.c2m_conv3x3_operand_f32(*args, None) == 1
        assert b'conv3x3_operand_f32: bad argument' in lib.c2m_last_error()
    assert lib.c2m_conv3x3_wgrad_scaled(p, p, p, p, p, None, 1, 8, 8, 18, 10, p, p, 1 << 20, None) == 1
    assert b'null x_amax' in lib.c2m_last_error()
    assert lib.c2m_conv3x3_wgrad_scaled(p, p, p, p, None, p, 1, 8, 8, 18, 10, p, p, 1 << 20, None) == 1
    assert b'null pointer' in lib.c2m_last_error()
    assert lib.c2m_conv3x3_wgrad_scaled(p, p, p, p, p, p, 0, 8, 8, 18, 10, p, p, 1 << 20, None) == 1
    assert b'bad shape' in lib.c2m_last_error()
    assert lib.c2m_conv3x3_wgrad_scaled(p, p, p, p, p, p, 1, 8, 8, 18, 9, p, p, 1 << 20, None) == 1
    assert b'smaller than one halo tile' in lib.c2m_last_error()
    a = _lib.ConvArgs()
    a.in_hi = a.in_lo = a.in2_hi = a.in2_lo = a.packed_w = a.out_f32 = a.x_amax = 16
    a.Cin, a.Cin2, a.B, a.H, a.W, a.Cout = 32, 8, 1, 18, 10, 8
    assert lib.c2m_conv3x3(ctypes.addressof(a), None) == 1
    assert b'single input' in lib.c2m_last_error()
    assert {'c2m_conv3x3_operand_f32', 'c2m_conv3x3_wgrad_scaled'} <= set(_lib.SYMBOLS)


def test_invalidate_packs_drops_the_dgrad_pack():
    from c2m_b200 import ops
    conv = torch.nn.Conv2d(8, 4, 3, 1, 1)
    for attr in ('_c2m_pack', '_c2m_pack_dgrad'):
        conv.weight.__dict__[attr] = ('tag', None, None, None)
    ops.invalidate_packs(conv)
    assert '_c2m_pack' not in conv.weight.__dict__ and '_c2m_pack_dgrad' not in conv.weight.__dict__
    w = torch.zeros(4, 8, 3, 3)
    w.__dict__['_c2m_pack_dgrad'] = ('tag', None, None, None)
    ops.invalidate_packs(w)
    assert '_c2m_pack_dgrad' not in w.__dict__


def test_routing_conv_is_nn_conv2d_off_the_gpu():
    """Same parameters, state-dict keys and gradients as nn.Conv2d when the tensor-core path does not apply."""
    from mmsr.models.archs.arch_util import Conv2d
    torch.manual_seed(0)
    ref = torch.nn.Conv2d(5, 7, 3, 1, 1)
    mine = Conv2d(5, 7, 3, 1, 1)
    mine.load_state_dict(ref.state_dict())
    assert isinstance(mine, torch.nn.Conv2d) and list(mine.state_dict()) == list(ref.state_dict())
    x = torch.randn(2, 5, 20, 12)
    for m in (ref, mine):
        F.leaky_relu(m(x), 0.1).square().sum().backward()
    assert torch.equal(ref.weight.grad, mine.weight.grad) and torch.equal(ref.bias.grad, mine.bias.grad)
