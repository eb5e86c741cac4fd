"""A/B of the general FFMA DCN forward (`c2m_deform_conv_forward_f32` with groups = 1, what `_ext.dcn_v2_forward`
runs under C2M_EXT_DCN_TC=0) between this tree's library and another build of it, e.g. the parent commit's:

    git worktree add /tmp/parent HEAD~1 && python /tmp/parent/c2-matching_b200/c2m_b200/build.py
    python tools/dcn_ffma_ab.py --other /tmp/parent/c2-matching_b200/lib/libc2m_sm100.so

Both libraries are loaded into one process and called on the same inputs, alternating A-B / B-A for --rounds rounds
of --reps calls each (CUDA events).  Workloads: BASELINE config 4 (64 -> 64, dg 8, 160^2) and the three restoration
DCN shapes (256 / 160^2, 128 / 320^2, 64 / 640^2; dg 8, B = 1), 3x3/s1/p1/d1, random offsets (std 2) and masks.
Prints the card, then per workload whether the outputs are bit-identical and each library's median / min / max ms.
Exits 1 if any output differs."""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200')]
import torch  # noqa: E402

SHAPES = (('config4_64_160', 64, 160), ('restoration_256_160', 256, 160), ('restoration_128_320', 128, 320),
          ('restoration_64_640', 64, 640))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--other', required=True, help='path of the other libc2m_sm100.so')
    ap.add_argument('--rounds', type=int, default=6)
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from c2m_b200 import _lib, ops
    libs = {'other': ctypes.CDLL(os.path.abspath(args.other)), 'this': ctypes.CDLL(_lib.LIB_PATH)}
    for lib in libs.values():
        lib.c2m_deform_conv_forward_f32.argtypes = _lib.SYMBOLS['c2m_deform_conv_forward_f32'][1]
    print(torch.cuda.get_device_name(0))
    dev, dg = 'cuda:0', 8
    gen = torch.Generator().manual_seed(3)
    same_all = True
    for name, C, H in SHAPES:
        x = torch.randn(1, C, H, H, generator=gen).to(dev)
        w = (torch.randn(C, C, 3, 3, generator=gen) * 0.05).to(dev)
        b = torch.randn(C, generator=gen).to(dev)
        off = (torch.randn(1, 18 * dg, H, H, generator=gen) * 2).to(dev)
        m = torch.rand(1, 9 * dg, H, H, generator=gen).to(dev)
        outs = {k: torch.empty(1, C, H, H, device=dev) for k in libs}
        s = ops._shape(x, C, 3, 3, 1, 1, 1, 1, 1, 1, dg, outs['this'])

        def run(k):
            rc = libs[k].c2m_deform_conv_forward_f32(x.data_ptr(), off.data_ptr(), m.data_ptr(), w.data_ptr(),
                                                     b.data_ptr(), 1, outs[k].data_ptr(), ctypes.byref(s),
                                                     ops._stream())
            if rc:
                raise RuntimeError(f'{k}: c2m_deform_conv_forward_f32 returned {rc}')
        for k in libs:
            for _ in range(3):
                run(k)
        times = {k: [] for k in libs}
        for r in range(args.rounds):
            for k in (list(libs) if r % 2 == 0 else list(libs)[::-1]):
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.reps):
                    run(k)
                e.record()
                e.synchronize()
                times[k].append(a.elapsed_time(e) / args.reps)
        same = torch.equal(outs['other'], outs['this'])
        same_all &= same
        stats = ', '.join(f'{k} median {sorted(v)[len(v) // 2]:.3f} ms (min {min(v):.3f}, max {max(v):.3f})'
                          for k, v in times.items())
        print(f'{name}: {"bit-identical" if same else "DIFFERENT"}; {stats}', flush=True)
    sys.exit(0 if same_all else 1)


if __name__ == '__main__':
    main()
