"""ORACLE — test infrastructure, NOT product code.

ctypes front-end for oracle/ordered_grad_oracle.c (the ordered input-gradient sums of deformable convolution and
deformable PS-ROI pooling, in the dtype).  `build()` compiles it with gcc into oracle/_build/ (git-ignored).  Takes and
returns CPU tensors; fp32 and fp64 run the matching C instantiation."""
import ctypes
import os
import subprocess

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'ordered_grad_oracle.c')
OUT_DIR = os.path.join(HERE, '_build')
LIB = os.path.join(OUT_DIR, 'libordered_grad_oracle.so')
_lib = None


def build(force=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    subprocess.run(['gcc', '-O2', '-ffp-contract=off', '-fPIC', '-shared', '-o', LIB, SRC, '-lm'], check=True)
    return LIB


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        _lib = ctypes.CDLL(LIB)
        for sfx in ('f32', 'f64'):
            getattr(_lib, f'oracle_deform_col2im_ordered_{sfx}').argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 13
            getattr(_lib, f'oracle_psroi_grad_input_ordered_{sfx}').argtypes = \
                [ctypes.c_void_p] * 4 + [ctypes.c_int] * 7 + [ctypes.c_float] + [ctypes.c_int] * 5 + \
                [ctypes.c_float, ctypes.c_void_p]
    return _lib


def _sfx(dtype):
    assert dtype in (torch.float32, torch.float64), dtype
    return 'f32' if dtype == torch.float32 else 'f64'


def _host(t, dtype):
    return None if t is None else t.detach().cpu().to(dtype).contiguous()


def deform_col2im(gcol, offset, mask, x_shape, kh, kw, sh, sw, ph, pw, dh, dw, dg):
    """gcol [B, C*kh*kw, Ho*Wo] (or any shape of that size) -> grad_input [B, C, H, W] in gcol's dtype, CPU.
    mask None is DCNv1 (modulation 1)."""
    dt = gcol.dtype
    gcol, offset, mask = [_host(t, dt) for t in (gcol, offset, mask)]
    B, C, H, W = x_shape
    gx = torch.empty(B, C, H, W, dtype=dt)
    rc = getattr(lib(), f'oracle_deform_col2im_ordered_{_sfx(dt)}')(
        gcol.data_ptr(), offset.data_ptr(), None if mask is None else mask.data_ptr(), gx.data_ptr(), B, C, H, W, kh,
        kw, sh, sw, ph, pw, dh, dw, dg)
    if rc:
        raise RuntimeError(f'oracle_deform_col2im_ordered rc={rc}')
    return gx


def psroi_grad_input(out_grad, x_shape, bbox, trans, top_count, no_trans, spatial_scale, output_dim, group_size,
                     pooled_size, part_size, sample_per_part, trans_std):
    """The `_ext.dcn_v2_psroi_pooling_backward` arguments with the input replaced by its shape -> grad_input
    [B, C, H, W] in out_grad's dtype, CPU."""
    dt = out_grad.dtype
    g, b, c = _host(out_grad, dt), _host(bbox, dt), _host(top_count, dt)
    t = None if no_trans else _host(trans, dt)
    K = 1 if no_trans else t.shape[1] // 2
    B, C, H, W = x_shape
    gx = torch.empty(B, C, H, W, dtype=dt)
    rc = getattr(lib(), f'oracle_psroi_grad_input_ordered_{_sfx(dt)}')(
        g.data_ptr(), b.data_ptr(), None if t is None else t.data_ptr(), c.data_ptr(), B, C, H, W, b.shape[0],
        int(bool(no_trans)), K, spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part,
        trans_std, gx.data_ptr())
    if rc:
        raise RuntimeError(f'oracle_psroi_grad_input_ordered rc={rc}')
    return gx
