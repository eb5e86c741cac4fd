"""ctypes binding of libc2m_sm100.so (the C ABI declared in include/c2m_sm100.h).

No fallback: if the library is missing or a call fails, this raises."""
import ctypes
import os

from .build import LIB_PATH

_lib = None

c_f32p = ctypes.c_void_p
c_i64p = ctypes.c_void_p


class DcnShape(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in
                ('B', 'C', 'H', 'W', 'Cout', 'kh', 'kw', 'sh', 'sw', 'ph', 'pw', 'dh', 'dw', 'dg')] + \
               [(n, ctypes.c_longlong) for n in
                ('xs_b', 'xs_c', 'xs_y', 'xs_x', 'os_b', 'os_c', 'os_y', 'os_x')]


class ConvArgs(ctypes.Structure):
    """c2m_conv3x3_args (include/c2m_sm100.h)."""
    _fields_ = [('in_hi', ctypes.c_void_p), ('in_lo', ctypes.c_void_p), ('Cin', ctypes.c_int),
                ('in2_hi', ctypes.c_void_p), ('in2_lo', ctypes.c_void_p), ('Cin2', ctypes.c_int),
                ('B', ctypes.c_int), ('H', ctypes.c_int), ('W', ctypes.c_int), ('sa_in', ctypes.c_int),
                ('packed_w', ctypes.c_void_p), ('bias', ctypes.c_void_p), ('Cout', ctypes.c_int), ('act', ctypes.c_int),
                ('res_hi', ctypes.c_void_p), ('res_lo', ctypes.c_void_p), ('res2_hi', ctypes.c_void_p),
                ('res2_lo', ctypes.c_void_p), ('sa_res', ctypes.c_int),
                ('out_hi', ctypes.c_void_p), ('out_lo', ctypes.c_void_p), ('sa_out', ctypes.c_int),
                ('pixel_shuffle', ctypes.c_int),
                ('out_f32', ctypes.c_void_p), ('add_f32', ctypes.c_void_p),
                ('os_b', ctypes.c_longlong), ('os_c', ctypes.c_longlong), ('os_y', ctypes.c_longlong),
                ('os_x', ctypes.c_longlong), ('out_f32_octets', ctypes.c_int), ('x_amax', ctypes.c_void_p)]


class DcnTcArgs(ctypes.Structure):
    """c2m_dcn_tc_args (include/c2m_sm100.h)."""
    _fields_ = [('x_il', ctypes.c_void_p),
                ('om', ctypes.c_void_p), ('pre', ctypes.c_void_p), ('idx', ctypes.c_void_p),
                ('gh', ctypes.c_int), ('gw', ctypes.c_int), ('ref_gw', ctypes.c_int), ('pre_scale', ctypes.c_int),
                ('B', ctypes.c_int), ('C', ctypes.c_int), ('H', ctypes.c_int), ('W', ctypes.c_int),
                ('Cout', ctypes.c_int), ('dg', ctypes.c_int),
                ('packed_w', ctypes.c_void_p), ('bias', ctypes.c_void_p), ('lrelu', ctypes.c_int),
                ('out_hi', ctypes.c_void_p), ('out_lo', ctypes.c_void_p), ('sa_out', ctypes.c_int),
                ('out_f32', ctypes.c_void_p), ('os_b', ctypes.c_longlong), ('os_c', ctypes.c_longlong),
                ('os_y', ctypes.c_longlong), ('os_x', ctypes.c_longlong), ('om_octets', ctypes.c_int),
                ('mask', ctypes.c_void_p), ('x_amax', ctypes.c_void_p), ('mask_amax', ctypes.c_void_p)]


class DcnTcGradArgs(ctypes.Structure):
    """c2m_dcn_tc_grad_args (include/c2m_sm100.h)."""
    _fields_ = [('gy_hi', ctypes.c_void_p), ('gy_lo', ctypes.c_void_p), ('gy_amax', ctypes.c_void_p),
                ('x_il', ctypes.c_void_p), ('x_amax', ctypes.c_void_p), ('mask_amax', ctypes.c_void_p),
                ('offset', ctypes.c_void_p), ('mask', ctypes.c_void_p)] + \
               [(n, ctypes.c_int) for n in ('B', 'C', 'H', 'W', 'Cout', 'dg')] + \
               [('packed_w', ctypes.c_void_p), ('grad_offset', ctypes.c_void_p), ('grad_mask', ctypes.c_void_p),
                ('grad_input', ctypes.c_void_p), ('grad_weight', ctypes.c_void_p), ('ws', ctypes.c_void_p),
                ('ws_bytes', ctypes.c_size_t)]


class PsroiShape(ctypes.Structure):
    """c2m_psroi_shape (include/c2m_sm100.h)."""
    _fields_ = [(n, ctypes.c_int) for n in ('B', 'C', 'H', 'W', 'R', 'no_trans', 'num_classes')] + \
               [('spatial_scale', ctypes.c_float), ('trans_std', ctypes.c_float)] + \
               [(n, ctypes.c_int) for n in ('output_dim', 'group_size', 'pooled_size', 'part_size', 'sample_per_part')]


_dshape = ctypes.POINTER(DcnShape)
_deform_fwd = (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int, ctypes.c_void_p, _dshape, ctypes.c_void_p])
_deform_im2col = (ctypes.c_int, [ctypes.c_void_p] * 3 + [_dshape, ctypes.c_void_p, ctypes.c_void_p])
_deform_coord = (ctypes.c_int, [ctypes.c_void_p] * 4 + [_dshape] + [ctypes.c_void_p] * 3)
_deform_col2im = (ctypes.c_int, [ctypes.c_void_p] * 3 + [_dshape, ctypes.c_void_p, ctypes.c_void_p])
_psroi_fwd = (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.POINTER(PsroiShape)] + [ctypes.c_void_p] * 3)
_psroi_bwd = (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.POINTER(PsroiShape)] + [ctypes.c_void_p] * 3 +
              [ctypes.c_size_t, ctypes.c_void_p])
_deform_col2im_det = (ctypes.c_int, [ctypes.c_void_p] * 3 + [_dshape] + [ctypes.c_void_p] * 2 +
                      [ctypes.c_size_t, ctypes.c_void_p])
_psroi_grad_det = (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.POINTER(PsroiShape)] + [ctypes.c_void_p] * 2 +
                   [ctypes.c_size_t, ctypes.c_void_p])

SYMBOLS = {
    'c2m_abi_version': (ctypes.c_int, []),
    'c2m_last_error': (ctypes.c_char_p, []),
    'c2m_launch_count': (ctypes.c_ulonglong, []),
    'c2m_conv3x3_packed_weight_bytes': (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    'c2m_conv3x3_pack_weights_f32': (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_psa_from_f32': (ctypes.c_int, [c_f32p] + [ctypes.c_int] * 4 + [ctypes.c_longlong] * 4 +
                         [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_psa_to_f32': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 + [c_f32p, c_f32p] +
                       [ctypes.c_longlong] * 4 + [ctypes.c_void_p]),
    'c2m_conv3x3': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_conv3x3_wgrad_workspace_bytes': (ctypes.c_size_t, [ctypes.c_int] * 5),
    'c2m_conv3x3_operand_f32': (ctypes.c_int, [c_f32p] + [ctypes.c_int] * 4 + [ctypes.c_longlong] * 4 +
                                [ctypes.c_void_p] * 4),
    'c2m_conv3x3_wgrad': (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int] * 5 +
                          [c_f32p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    'c2m_conv3x3_wgrad_scaled': (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int] * 5 +
                                 [c_f32p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    'c2m_psa_maxpool2': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 3),
    'c2m_dcn_tc_supported': (ctypes.c_int, [ctypes.c_int] * 3),
    'c2m_dcn_tc_packed_weight_bytes': (ctypes.c_size_t, [ctypes.c_int] * 3),
    'c2m_dcn_tc_pack_weights_f32': (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_dcn_v2_fused_tc': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_dcn_tc_operand_bytes': (ctypes.c_size_t, [ctypes.c_int] * 5),
    'c2m_dcn_tc_operand_psa': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 +
                               [ctypes.c_void_p] * 2),
    'c2m_dcn_tc_operand_f32': (ctypes.c_int, [c_f32p] + [ctypes.c_int] * 4 + [ctypes.c_longlong] * 4 +
                               [ctypes.c_int, c_f32p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_dcn_tc_dgrad_packed_weight_bytes': (ctypes.c_size_t, [ctypes.c_int] * 3),
    'c2m_dcn_tc_pack_dgrad_weights_f32': (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                         ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_dcn_tc_dgrad': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_dcn_tc_wgrad_workspace_bytes': (ctypes.c_size_t, [ctypes.c_int] * 6),
    'c2m_dcn_tc_wgrad': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    'c2m_profile_enable': (ctypes.c_int, [ctypes.c_int]),
    'c2m_profile_collect': (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int),
                                           ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]),
    'c2m_corr_workspace_bytes': (ctypes.c_size_t, [ctypes.c_int] * 9),
    'c2m_corr_argmax_f32': (ctypes.c_int, [c_f32p, c_f32p] + [ctypes.c_int] * 12 + [ctypes.c_uint, c_i64p, c_f32p,
                                                                                 ctypes.c_void_p, ctypes.c_size_t,
                                                                                 ctypes.c_void_p]),
    'c2m_offset_pyramid_f32': (ctypes.c_int, [c_i64p] + [ctypes.c_int] * 5 + [c_f32p, ctypes.c_void_p]),
    'c2m_dcn_v2_fused_forward_f32': (ctypes.c_int, [c_f32p, c_f32p, c_f32p, c_i64p] + [ctypes.c_int] * 4 +
                                     [c_f32p, c_f32p, ctypes.c_float, c_f32p, ctypes.POINTER(DcnShape),
                                      ctypes.c_void_p]),
    'c2m_psroi_pooling_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(PsroiShape), ctypes.c_int]),
    'c2m_psroi_pooling_forward_f32': _psroi_fwd,
    'c2m_psroi_pooling_forward_f64': _psroi_fwd,
    'c2m_psroi_pooling_backward_f32': _psroi_bwd,
    'c2m_psroi_pooling_backward_f64': _psroi_bwd,
    'c2m_deform_conv_forward_f32': _deform_fwd,
    'c2m_deform_conv_forward_f64': _deform_fwd,
    'c2m_deform_conv_im2col_f32': _deform_im2col,
    'c2m_deform_conv_im2col_f64': _deform_im2col,
    'c2m_deform_conv_col2im_coord_f32': _deform_coord,
    'c2m_deform_conv_col2im_coord_f64': _deform_coord,
    'c2m_deform_conv_col2im_f32': _deform_col2im,
    'c2m_deform_conv_col2im_f64': _deform_col2im,
    'c2m_dcn_col2im_det_workspace_bytes': (ctypes.c_size_t, [_dshape, ctypes.c_int]),
    'c2m_deform_conv_col2im_det_f32': _deform_col2im_det,
    'c2m_deform_conv_col2im_det_f64': _deform_col2im_det,
    'c2m_psroi_grad_input_det_workspace_bytes': (ctypes.c_size_t, [ctypes.POINTER(PsroiShape), ctypes.c_int]),
    'c2m_psroi_pooling_grad_input_det_f32': _psroi_grad_det,
    'c2m_psroi_pooling_grad_input_det_f64': _psroi_grad_det,
}


class C2MError(RuntimeError):
    pass


EXPECTED_ABI = 7      # c2m_abi_version() the ctypes structs above mirror (include/c2m_sm100.h)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise C2MError(
                f'{LIB_PATH} not built: run `python -c "import __graft_entry__ as g; g.build()"` '
                '(no CPU/PyTorch fallback exists for the H100 hot path)')
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(l, name)          # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        got = l.c2m_abi_version()
        if got != EXPECTED_ABI:
            raise C2MError(f'{LIB_PATH} has ABI version {got}, these bindings are written for {EXPECTED_ABI}: '
                           'rebuild it (python -c "import __graft_entry__ as g; g.build()")')
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().c2m_last_error().decode(errors='replace')
        raise C2MError(f'{what} failed (status {rc}): {msg}')


def check_size(nbytes, what):
    """The byte count a size query returned; 0 means the query failed."""
    if nbytes == 0:
        raise C2MError(f'{what}: ' + lib().c2m_last_error().decode(errors='replace'))
    return nbytes
