"""The `mmsr.models.archs.dcn` drop-in without a GPU: the package surface, the `deform_conv_cuda` functions with the
reference's positional order, constructor signatures, parameter shapes, initialisation and state-dict keys, and the
errors raised before any kernel launch (CPU tensors, fp16, 3-D input, output channels not divisible by groups)."""
import inspect

import pytest
import torch

DCN_NAMES = ['DeformConv', 'DeformConvPack', 'ModulatedDeformConv', 'ModulatedDeformConvPack', 'deform_conv',
             'modulated_deform_conv']

# deform_conv_cuda.cpp:151-573 (the pybind export at :681-695)
CUDA_FUNCTIONS = {
    'deform_conv_forward_cuda': 'input weight offset output columns ones kW kH dW dH padW padH dilationW dilationH '
                                'group deformable_group im2col_step',
    'deform_conv_backward_input_cuda': 'input offset gradOutput gradInput gradOffset weight columns kW kH dW dH padW '
                                       'padH dilationW dilationH group deformable_group im2col_step',
    'deform_conv_backward_parameters_cuda': 'input offset gradOutput gradWeight columns ones kW kH dW dH padW padH '
                                            'dilationW dilationH group deformable_group scale im2col_step',
    'modulated_deform_conv_cuda_forward': 'input weight bias ones offset mask output columns kernel_h kernel_w '
                                          'stride_h stride_w pad_h pad_w dilation_h dilation_w group deformable_group '
                                          'with_bias',
    'modulated_deform_conv_cuda_backward': 'input weight bias ones offset mask columns grad_input grad_weight '
                                           'grad_bias grad_offset grad_mask grad_output kernel_h kernel_w stride_h '
                                           'stride_w pad_h pad_w dilation_h dilation_w group deformable_group '
                                           'with_bias',
}


def test_dcn_package_surface():
    import mmsr.models.archs.dcn as dcn
    assert sorted(dcn.__all__) == sorted(DCN_NAMES)
    for n in DCN_NAMES:
        assert hasattr(dcn, n), n


def test_deform_conv_cuda_functions_keep_reference_argument_order():
    from mmsr.models.archs.dcn import deform_conv_cuda
    for name, params in CUDA_FUNCTIONS.items():
        assert list(inspect.signature(getattr(deform_conv_cuda, name)).parameters) == params.split(), name


def test_constructor_signatures():
    from mmsr.models.archs.dcn import DeformConv, ModulatedDeformConv, ModulatedDeformConvPack
    want = ['in_channels', 'out_channels', 'kernel_size', 'stride', 'padding', 'dilation', 'groups',
            'deformable_groups', 'bias']
    for cls, bias_default in ((DeformConv, False), (ModulatedDeformConv, True)):
        sig = inspect.signature(cls.__init__)
        assert list(sig.parameters)[1:] == want, cls
        d = {k: v.default for k, v in sig.parameters.items()}
        assert (d['stride'], d['padding'], d['dilation'], d['groups'], d['deformable_groups'], d['bias']) == \
            (1, 0, 1, 1, 1, bias_default), cls
    m = ModulatedDeformConvPack(4, 4, 3, padding=1, extra_offset_mask=True)
    assert m.extra_offset_mask and m.debug_offset_check is False
    with pytest.raises(AssertionError):
        DeformConv(4, 4, 3, bias=True)
    with pytest.raises(AssertionError):
        DeformConv(6, 4, 3, groups=4)


def test_state_dict_keys_shapes_and_init():
    from mmsr.models.archs.dcn import DeformConv, DeformConvPack, ModulatedDeformConv, ModulatedDeformConvPack
    shapes = lambda m: {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes(DeformConv(6, 8, (3, 5), groups=2)) == {'weight': (8, 3, 3, 5)}
    assert shapes(DeformConvPack(6, 8, 3, padding=1, groups=2, deformable_groups=3)) == {
        'weight': (8, 3, 3, 3), 'conv_offset.weight': (54, 6, 3, 3), 'conv_offset.bias': (54,)}
    assert shapes(ModulatedDeformConv(4, 6, 3, groups=2, bias=False)) == {'weight': (6, 2, 3, 3)}
    m = ModulatedDeformConvPack(8, 4, 3, padding=1, deformable_groups=2)
    assert shapes(m) == {'weight': (4, 8, 3, 3), 'bias': (4,), 'conv_offset_mask.weight': (54, 8, 3, 3),
                         'conv_offset_mask.bias': (54,)}
    bound = 1 / (8 * 9) ** 0.5            # n counts every input channel, also with groups
    wmax = float(m.weight.detach().abs().max())
    assert 0.5 * bound < wmax <= bound
    assert not m.bias.any() and not m.conv_offset_mask.weight.any() and not m.conv_offset_mask.bias.any()
    g = ModulatedDeformConv(8, 4, 3, groups=4)
    assert float(g.weight.detach().abs().max()) <= bound


def _args(dtype=torch.float32, cout=4, groups=1, dim=4):
    x = torch.zeros(2, 4, 7, 7, dtype=dtype)
    if dim == 3:
        x = x[0]
    return x, torch.zeros(2, 18, 5, 5, dtype=dtype), torch.ones(2, 9, 5, 5, dtype=dtype), \
        torch.zeros(cout, 4 // groups, 3, 3, dtype=dtype)


def test_cpu_tensors_raise():
    from mmsr.models.archs.dcn import deform_conv, deform_conv_cuda, modulated_deform_conv
    from c2m_b200 import ops
    x, off, mask, w = _args()
    with pytest.raises(NotImplementedError):
        deform_conv(x, off, w)
    with pytest.raises(NotImplementedError):
        modulated_deform_conv(x, off, mask, w)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        deform_conv_cuda.deform_conv_forward_cuda(x, w, off, torch.empty(2, 4, 5, 5), None, None,
                                                  3, 3, 1, 1, 0, 0, 1, 1, 1, 1, 2)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        ops.deform_conv_backward(x, w, off, mask, torch.zeros(2, 4, 5, 5), 3, 3, 1, 1, 0, 0, 1, 1, 1, 1)


def test_fp16_raises():
    from c2m_b200 import ops
    x, off, mask, w = _args(torch.float16)
    with pytest.raises(RuntimeError, match='float32 and torch.float64'):
        ops.deform_conv_forward(x, w, off, mask, None, 3, 3, 1, 1, 0, 0, 1, 1, 1, 1)
    with pytest.raises(RuntimeError, match='float32 and torch.float64'):
        ops.deform_conv_backward(x, w, off, None, torch.zeros(2, 4, 5, 5, dtype=torch.float16),
                                 3, 3, 1, 1, 0, 0, 1, 1, 1, 1)


def test_3d_input_raises():
    from mmsr.models.archs.dcn import deform_conv, deform_conv_cuda, modulated_deform_conv
    x, off, mask, w = _args(dim=3)
    with pytest.raises(ValueError, match='Expected 4D tensor'):
        deform_conv(x, off[0], w)
    with pytest.raises(ValueError, match='Expected 4D tensor'):
        modulated_deform_conv(x, off[0], mask[0], w)
    with pytest.raises(RuntimeError, match='4D input'):
        deform_conv_cuda.modulated_deform_conv_cuda_forward(x, w, None, None, off[0], mask[0], None, None,
                                                            3, 3, 1, 1, 0, 0, 1, 1, 1, 1, False)


def test_cout_not_divisible_by_groups_raises():
    from c2m_b200 import ops
    x, off, mask, w = _args(cout=3, groups=2)
    with pytest.raises(RuntimeError, match=r'output channels \(3\) must be divisible by groups \(2\)'):
        ops.deform_conv_forward(x, w, off, mask, None, 3, 3, 1, 1, 0, 0, 1, 1, 2, 1)


def test_modulated_boundary_keeps_contiguity_errors():
    from mmsr.models.archs.dcn import deform_conv_cuda
    x, off, mask, w = _args()
    with pytest.raises(RuntimeError, match='input tensor has to be contiguous'):
        deform_conv_cuda.modulated_deform_conv_cuda_forward(x.transpose(2, 3), w, None, None, off, mask, None, None,
                                                            3, 3, 1, 1, 0, 0, 1, 1, 1, 1, False)
    with pytest.raises(RuntimeError, match='weight tensor has to be contiguous'):
        deform_conv_cuda.modulated_deform_conv_cuda_backward(x, w.transpose(2, 3), None, None, off, mask, None, None,
                                                             None, None, None, None, None, 3, 3, 1, 1, 0, 0, 1, 1,
                                                             1, 1, False)


def test_library_rejects_bad_groups_before_launch():
    """The library validates groups itself (no device needed: the check precedes any CUDA call)."""
    import ctypes
    import __graft_entry__ as g
    g.build()
    from c2m_b200 import _lib
    L = _lib.lib()
    s = _lib.DcnShape(B=1, C=6, H=5, W=5, Cout=4, kh=3, kw=3, sh=1, sw=1, ph=0, pw=0, dh=1, dw=1, dg=1,
                      xs_b=150, xs_c=25, xs_y=5, xs_x=1, os_b=36, os_c=9, os_y=3, os_x=1)
    dummy = ctypes.c_void_p(16)
    for groups, what in ((3, b'divisible by groups'), (0, b'divisible by groups'), (4, b'divisible by groups')):
        rc = L.c2m_deform_conv_forward_f64(dummy, dummy, None, dummy, None, groups, dummy, s, None)
        assert rc == 1 and what in L.c2m_last_error(), groups
    rc = L.c2m_deform_conv_col2im_coord_f32(dummy, dummy, dummy, dummy, s, dummy, None, None)
    assert rc == 1 and b'grad_mask must be given exactly when mask is' in L.c2m_last_error()
