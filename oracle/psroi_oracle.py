"""ORACLE — test infrastructure, NOT product code.

ctypes front-end for oracle/psroi_oracle.c (the literal plain-C restatement of deformable PS-ROI pooling).  `build()`
compiles it with gcc into oracle/_build/ (git-ignored).  Takes and returns CPU tensors; fp32 and fp64 run the matching
C instantiation.  The argument lists are those of `_ext.dcn_v2_psroi_pooling_forward` / `_backward`."""
import ctypes
import os
import subprocess

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'psroi_oracle.c')
OUT_DIR = os.path.join(HERE, '_build')
LIB = os.path.join(OUT_DIR, 'libpsroi_oracle.so')
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
            getattr(_lib, f'oracle_psroi_forward_{sfx}').argtypes = \
                [ctypes.c_void_p] * 3 + [ctypes.c_int] * 7 + [ctypes.c_float] + [ctypes.c_int] * 5 + \
                [ctypes.c_float] + [ctypes.c_void_p] * 2
            getattr(_lib, f'oracle_psroi_backward_{sfx}').argtypes = \
                [ctypes.c_void_p] * 5 + [ctypes.c_int] * 7 + [ctypes.c_float] + [ctypes.c_int] * 5 + \
                [ctypes.c_float] + [ctypes.c_void_p] * 2
    return _lib


def _prep(input, bbox, trans, no_trans):
    dt = input.dtype
    assert dt in (torch.float32, torch.float64), dt
    x = input.detach().cpu().contiguous()
    b = bbox.detach().cpu().to(dt).contiguous()
    t = None if no_trans else trans.detach().cpu().to(dt).contiguous()
    K = 1 if no_trans else t.shape[1] // 2
    return x, b, t, K, 'f32' if dt == torch.float32 else 'f64'


def forward(input, bbox, trans, no_trans, spatial_scale, output_dim, group_size, pooled_size, part_size,
            sample_per_part, trans_std):
    """-> (output, output_count) [R, output_dim, P, P], CPU, input's dtype."""
    x, b, t, K, sfx = _prep(input, bbox, trans, no_trans)
    B, C, H, W = x.shape
    R = b.shape[0]
    out = torch.empty(R, output_dim, pooled_size, pooled_size, dtype=x.dtype)
    cnt = torch.empty_like(out)
    rc = getattr(lib(), f'oracle_psroi_forward_{sfx}')(
        x.data_ptr(), b.data_ptr(), None if t is None else t.data_ptr(), B, C, H, W, R, int(bool(no_trans)), K,
        spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part, trans_std,
        out.data_ptr(), cnt.data_ptr())
    if rc:
        raise RuntimeError(f'oracle_psroi_forward_{sfx} rc={rc}')
    return out, cnt


def backward(out_grad, input, bbox, trans, top_count, no_trans, spatial_scale, output_dim, group_size, pooled_size,
             part_size, sample_per_part, trans_std):
    """-> (grad_input, grad_trans), CPU, input's dtype; grad_trans is zeros_like(trans) when no_trans."""
    x, b, t, K, sfx = _prep(input, bbox, trans, no_trans)
    B, C, H, W = x.shape
    R = b.shape[0]
    g = out_grad.detach().cpu().to(x.dtype).contiguous()
    c = top_count.detach().cpu().to(x.dtype).contiguous()
    gx = torch.empty_like(x)
    gt = torch.zeros_like(trans.detach().cpu()) if no_trans else torch.empty_like(t)
    rc = getattr(lib(), f'oracle_psroi_backward_{sfx}')(
        g.data_ptr(), x.data_ptr(), b.data_ptr(), None if t is None else t.data_ptr(), c.data_ptr(), B, C, H, W, R,
        int(bool(no_trans)), K, spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part,
        trans_std, gx.data_ptr(), None if no_trans else gt.data_ptr())
    if rc:
        raise RuntimeError(f'oracle_psroi_backward_{sfx} rc={rc}')
    return gx, gt
