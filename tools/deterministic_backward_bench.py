"""Backward device time with torch's deterministic algorithms off (atomic grad_input scatter) and on (ordered
grad_input gather), CUDA events, the two modes alternated call by call, median of --iters calls after --warmup calls.

Workloads: the four of tools/deform_conv_bench.py (autograd backward of every gradient), the three of
tools/psroi_bench.py (`_ext.dcn_v2_psroi_pooling_backward`), and `_ext.dcn_v2_backward` on the three restoration DCN
shapes (256 ch at 160x160, 128 at 320x320, 64 at 640x640, dg 8, B = 1).  Prints the card name and power limit read in
the same run, one line per workload, and the largest ordered-gather workspace allocated.

    CUBLAS_WORKSPACE_CONFIG=:4096:8 python tools/deterministic_backward_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tools')]
os.environ.setdefault('CUBLAS_WORKSPACE_CONFIG', ':4096:8')
import torch  # noqa: E402

import deform_conv_bench as dcb  # noqa: E402
import psroi_bench as psb  # noqa: E402

RESTORATION = {'ext_256_160x160_dg8': (256, 160), 'ext_128_320x320_dg8': (128, 320), 'ext_64_640x640_dg8': (64, 640)}


def alternate(fn, iters, warmup):
    """Median ms of fn() with deterministic algorithms off and on, alternating call by call."""
    ts = {False: [], True: []}
    for i in range(warmup + iters):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if i >= warmup:
                ts[det].append(a.elapsed_time(b))
    torch.use_deterministic_algorithms(False)
    return [sorted(ts[d])[len(ts[d]) // 2] for d in (False, True)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import _ext
    from c2m_b200 import ops
    from mmsr.models.archs.dcn import deform_conv, modulated_deform_conv
    torch.backends.cuda.matmul.allow_tf32 = False
    print(dcb.card())
    dev = 'cuda:0'
    rows = []

    for name, (B, C, Cout, groups, dg, H, W, modulated) in dcb.WORKLOADS.items():
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(B, C, H, W, device=dev, generator=gen).requires_grad_(True)
        w = (torch.randn(Cout, C // groups, 3, 3, device=dev, generator=gen) * 0.05).requires_grad_(True)
        off = (torch.randn(B, 18 * dg, H, W, device=dev, generator=gen) * 2.0).requires_grad_(True)
        mask = torch.rand(B, 9 * dg, H, W, device=dev, generator=gen).requires_grad_(True) if modulated else None
        bias = torch.zeros(Cout, device=dev, requires_grad=True) if modulated else None
        gout = torch.randn(B, Cout, H, W, device=dev, generator=gen)
        leaves = [t for t in (x, w, off, mask, bias) if t is not None]
        y = (modulated_deform_conv(x, off, mask, w, bias, 1, 1, 1, groups, dg) if modulated
             else deform_conv(x, off, w, 1, 1, 1, groups, dg))
        rows.append((f'deform_conv {name}', alternate(lambda: torch.autograd.grad(y, leaves, gout, retain_graph=True),
                                                      args.iters, args.warmup)))

    for name, (B, C, H, W, R, P, S, scale, tstd, side) in psb.WORKLOADS.items():
        x, rois, trans = psb.inputs(B, C, H, W, R, P, scale, side)
        a = (False, scale, C, 1, P, P, S, tstd)
        out, cnt = _ext.dcn_v2_psroi_pooling_forward(x, rois, trans, *a)
        gout = torch.randn_like(out)
        rows.append((f'psroi {name}', alternate(lambda: _ext.dcn_v2_psroi_pooling_backward(gout, x, rois, trans, cnt,
                                                                                          *a), args.iters,
                                                args.warmup)))

    for name, (C, S) in RESTORATION.items():
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(1, C, S, S, device=dev, generator=gen)
        w = torch.randn(C, C, 3, 3, device=dev, generator=gen) * 0.05
        b = torch.zeros(C, device=dev)
        off = torch.randn(1, 144, S, S, device=dev, generator=gen) * 2.0
        mask = torch.rand(1, 72, S, S, device=dev, generator=gen)
        gout = torch.randn(1, C, S, S, device=dev, generator=gen)
        rows.append((f'_ext.dcn_v2_backward {name}',
                     alternate(lambda: _ext.dcn_v2_backward(x, w, b, off, mask, gout, 3, 3, 1, 1, 1, 1, 1, 1, 8),
                               args.iters, args.warmup)))

    for name, (off_ms, on_ms) in rows:
        print(f'{name} | atomic {off_ms:.3f} ms | ordered {on_ms:.3f} ms | ordered / atomic {on_ms / off_ms:.2f}',
              flush=True)
    print(f'peak ordered-gather workspace {ops.det_workspace_peak / 2**20:.1f} MiB')


if __name__ == '__main__':
    main()
