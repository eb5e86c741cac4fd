"""Deformable PS-ROI pooling (`_ext.dcn_v2_psroi_pooling_forward` / `_backward`): device time of the forward and the
backward with CUDA events, and torchvision's roi_align on the same ROIs as a yardstick.

roi_align (sampling_ratio=S, aligned=False) is a DIFFERENT op: it averages S x S samples at sub-bin centres per bin
and never drops a sample.  It reads the same number of bilinear samples (R * C * P^2 * S^2, four corners each), so its
rate says how fast this hardware gathers that many samples through a mature kernel.

Workloads: (a) the reference DCNv2 README example (B=2, C=32, 64x64, 20 ROIs, P=7, S=4, scale 1/4): overhead;
(b) detector-sized: B=2, C=256, 50x76 at scale 1/16, 512 ROIs, P=7, S=4, part 7, trans_std 0.1; (c) the same on a
200x304 map at scale 1/4.  Prints the card name and power limit read in the same run, then one line per workload.

    python tools/psroi_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200')]
import torch  # noqa: E402

WORKLOADS = {   # name: (B, C, H, W, R, P, S, scale, trans_std, roi side range in image pixels)
    'a_readme': (2, 32, 64, 64, 20, 7, 4, 1 / 4, 0.1, (1, 64)),
    'b_detector_1/16': (2, 256, 50, 76, 512, 7, 4, 1 / 16, 0.1, (32, 512)),
    'c_detector_1/4': (2, 256, 200, 304, 512, 7, 4, 1 / 4, 0.1, (32, 512)),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = 'power limit not readable'
    return f'{name}, {q}'


def inputs(B, C, H, W, R, P, scale, side, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g)
    iw, ih = W / scale, H / scale
    wh = torch.randint(side[0], side[1], (R, 2), generator=g).float()
    xy = torch.rand(R, 2, generator=g) * (torch.tensor([iw, ih]) - wh).clamp(min=1)
    b = torch.randint(0, B, (R, 1), generator=g).float()
    rois = torch.cat([b, xy, xy + wh], 1)
    trans = torch.randn(R, 2, P, P, generator=g)
    return x.cuda(), rois.cuda(), trans.cuda()


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('psroi_bench: no CUDA device')
    import _ext
    from torchvision.ops import roi_align
    print(f'card: {card()}')
    print('workload | samples | fwd ms (median, min) | fwd Gsamples/s | bwd ms (median, min) | '
          'roi_align ms (median, min) [different op] | roi_align Gsamples/s | fwd / roi_align')
    for name, (B, C, H, W, R, P, S, scale, tstd, side) in WORKLOADS.items():
        x, rois, trans = inputs(B, C, H, W, R, P, scale, side)
        args = (0, scale, C, 1, P, P, S, tstd)
        out, cnt = _ext.dcn_v2_psroi_pooling_forward(x, rois, trans, *args)
        gout = torch.randn_like(out)
        fwd = time_ms(lambda: _ext.dcn_v2_psroi_pooling_forward(x, rois, trans, *args), a.iters, a.warmup)
        bwd = time_ms(lambda: _ext.dcn_v2_psroi_pooling_backward(gout, x, rois, trans, cnt, *args), a.iters, a.warmup)
        ra = time_ms(lambda: roi_align(x, rois, P, spatial_scale=scale, sampling_ratio=S, aligned=False), a.iters,
                     a.warmup)
        n = R * C * P * P * S * S
        print(f'{name} | {n} | {fwd[0]:.4f}, {fwd[1]:.4f} | {n / fwd[0] / 1e6:.1f} | {bwd[0]:.4f}, {bwd[1]:.4f} | '
              f'{ra[0]:.4f}, {ra[1]:.4f} | {n / ra[0] / 1e6:.1f} | {fwd[0] / ra[0]:.2f}')


if __name__ == '__main__':
    main()
