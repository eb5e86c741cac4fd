"""Grouped deformable convolution (`mmsr.models.archs.dcn`): device time of the forward and of the backward (all
gradients), fp32, CUDA events, median over --iters calls after --warmup calls, next to torchvision's
`deform_conv2d` on CUDA with the same inputs (the same op: conv groups through the weight shape, optional mask).

Workloads: (a) v1, B = 2, 512 -> 512, 3x3, 25x38 (a ResNet C5-style DCN); (b) modulated, 256 -> 256, dg = 4, 100x152;
(c) grouped, 256 -> 256, groups = 32, dg = 4, 50x76; (d) modulated, 64 -> 64, dg = 8, 180x320 (the tensor-core
route).  B = 1 unless stated, stride 1, padding 1.  Prints the card name and power limit read in the same run, then
one line per workload.

    python tools/deform_conv_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200')]
import torch  # noqa: E402

WORKLOADS = {   # name: (B, C, Cout, groups, dg, H, W, modulated)
    'a_v1_512_25x38': (2, 512, 512, 1, 1, 25, 38, False),
    'b_mod_256_dg4_100x152': (1, 256, 256, 1, 4, 100, 152, True),
    'c_grouped_256_g32_dg4_50x76': (1, 256, 256, 32, 4, 50, 76, True),
    'd_mod_64_dg8_180x320_tc': (1, 64, 64, 1, 8, 180, 320, True),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = 'power limit not readable'
    return f'{name}, {q}'


def timed(fn, iters, warmup):
    """Median device time in ms of fn() over `iters` calls, each bracketed by its own pair of events."""
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from torchvision.ops import deform_conv2d
    from mmsr.models.archs.dcn import deform_conv, modulated_deform_conv
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    print(card())
    dev = 'cuda:0'
    for name, (B, C, Cout, groups, dg, H, W, modulated) in WORKLOADS.items():
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(B, C, H, W, device=dev, generator=gen).requires_grad_(True)
        w = (torch.randn(Cout, C // groups, 3, 3, device=dev, generator=gen) * 0.05).requires_grad_(True)
        off = (torch.randn(B, 18 * dg, H, W, device=dev, generator=gen) * 2.0).requires_grad_(True)
        mask = torch.rand(B, 9 * dg, H, W, device=dev, generator=gen).requires_grad_(True) if modulated else None
        bias = torch.zeros(Cout, device=dev, requires_grad=True) if modulated else None
        gout = torch.randn(B, Cout, H, W, device=dev, generator=gen)
        leaves = [t for t in (x, w, off, mask, bias) if t is not None]

        def ours():
            if modulated:
                return modulated_deform_conv(x, off, mask, w, bias, 1, 1, 1, groups, dg)
            return deform_conv(x, off, w, 1, 1, 1, groups, dg)

        def tv():
            return deform_conv2d(x, off, w, bias, stride=1, padding=1, dilation=1, mask=mask)

        row = [name]
        for label, fn in (('ours', ours), ('torchvision', tv)):
            with torch.no_grad():
                fwd = timed(fn, args.iters, args.warmup)
            y = fn()

            def bwd():
                torch.autograd.grad(y, leaves, gout, retain_graph=True)
            row.append(f'{label} fwd {fwd:.3f} ms bwd {timed(bwd, args.iters, args.warmup):.3f} ms')
        with torch.no_grad():
            err = float((ours() - tv()).abs().max() / tv().abs().max())
        row.append(f'max |ours - torchvision| / scale {err:.1e}')
        print(' | '.join(row), flush=True)


if __name__ == '__main__':
    main()
