"""ORACLE — test infrastructure, NOT product code.

ctypes front-end for oracle/deform_conv_oracle.c (the literal plain-C restatement of grouped deformable convolution,
v1 and modulated).  `build()` compiles it with gcc into oracle/_build/ (git-ignored).  Takes and returns CPU tensors;
fp32 and fp64 run the matching C instantiation.  mask None is DCNv1 (modulation 1), bias None adds nothing."""
import ctypes
import os
import subprocess

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'deform_conv_oracle.c')
OUT_DIR = os.path.join(HERE, '_build')
LIB = os.path.join(OUT_DIR, 'libdeform_conv_oracle.so')
_lib = None


def build(force=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    subprocess.run(['gcc', '-O2', '-fopenmp', '-ffp-contract=off', '-fPIC', '-shared', '-o', LIB, SRC, '-lm'],
                   check=True)
    return LIB


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        _lib = ctypes.CDLL(LIB)
        for sfx in ('f32', 'f64'):
            getattr(_lib, f'oracle_deform_conv_forward_{sfx}').argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int] * 15
            getattr(_lib, f'oracle_deform_conv_backward_{sfx}').argtypes = [ctypes.c_void_p] * 10 + [ctypes.c_int] * 15
    return _lib


def _host(t, dtype):
    return None if t is None else t.detach().cpu().to(dtype).contiguous()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _sfx(dtype):
    assert dtype in (torch.float32, torch.float64), dtype
    return 'f32' if dtype == torch.float32 else 'f64'


def out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw):
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def forward(x, weight, bias, offset, mask, kh, kw, sh, sw, ph, pw, dh, dw, groups, dg):
    """-> out [B, Cout, Ho, Wo], CPU, x's dtype."""
    dt = x.dtype
    x, weight, bias, offset, mask = [_host(t, dt) for t in (x, weight, bias, offset, mask)]
    B, C, H, W = x.shape
    cout = weight.shape[0]
    out = torch.empty(B, cout, *out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw), dtype=dt)
    rc = getattr(lib(), f'oracle_deform_conv_forward_{_sfx(dt)}')(
        _ptr(x), _ptr(weight), _ptr(bias), _ptr(offset), _ptr(mask), _ptr(out), B, C, H, W, cout, kh, kw, sh, sw, ph,
        pw, dh, dw, groups, dg)
    if rc:
        raise RuntimeError(f'oracle_deform_conv_forward rc={rc}')
    return out


def backward(x, weight, offset, mask, grad_output, kh, kw, sh, sw, ph, pw, dh, dw, groups, dg):
    """-> (grad_input, grad_offset, grad_mask or None, grad_weight, grad_bias), CPU, x's dtype."""
    dt = x.dtype
    x, weight, offset, mask, gout = [_host(t, dt) for t in (x, weight, offset, mask, grad_output)]
    B, C, H, W = x.shape
    cout = weight.shape[0]
    gx, goff, gw = torch.empty_like(x), torch.empty_like(offset), torch.empty_like(weight)
    gm = torch.empty_like(mask) if mask is not None else None
    gb = torch.empty(cout, dtype=dt)
    rc = getattr(lib(), f'oracle_deform_conv_backward_{_sfx(dt)}')(
        _ptr(x), _ptr(weight), _ptr(offset), _ptr(mask), _ptr(gout), _ptr(gx), _ptr(goff), _ptr(gm), _ptr(gw),
        _ptr(gb), B, C, H, W, cout, kh, kw, sh, sw, ph, pw, dh, dw, groups, dg)
    if rc:
        raise RuntimeError(f'oracle_deform_conv_backward rc={rc}')
    return gx, goff, gm, gw, gb
