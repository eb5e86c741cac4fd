"""Backward of the 3x3 convolution: device time of dX and dW on the tensor-core path (ops.conv3x3's backward) next to
cuDNN fp32 with TF32 off and with TF32 on, and one RestorationNet forward + backward on each path.

Shapes are the stage-3 training step of options/train/stage3_restoration_mse.yml (batch 9, GT 160: LR 40, 64-channel maps
at 40x40, 80x80 and 160x160): the ResBlock convolutions, the concatenating head_* and *_offset_conv1 layers
(64 + C) -> 64 and (64 + C) -> C for C = 256, 128, 64, conv_offset_mask C -> 216, the tails 64 -> 256, 64 -> 32 and
32 -> 3, and conv_first 3 -> 64.  Tensor-core dX = grad_output -> PSA (amax and conversion) + the 3x3 kernel with the
rotated weights + unscale; dW = conv3x3_wgrad_kernel + its ordered reduction (given the PSA operands, which the
backward shares with dX; the conversion is listed on its own).  cuDNN: torch.nn.grad.conv2d_input / conv2d_weight.
CUDA events, median over --iters calls after --warmup.  Prints the card name and power limit read in the same run, one
line per shape and the net_g step; with --out FILE it also writes everything there as JSON.

    python tools/conv_backward_bench.py [--iters 20] [--warmup 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')]
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

B = 9
SHAPES = [   # (name, Cin, Cout, H)
    ('resblock_40', 64, 64, 40), ('resblock_80', 64, 64, 80), ('resblock_160', 64, 64, 160),
    ('head_small', 320, 64, 40), ('offset_conv1_small', 320, 256, 40),
    ('head_medium', 192, 64, 80), ('offset_conv1_medium', 192, 128, 80),
    ('head_large', 128, 64, 160), ('offset_conv1_large', 128, 64, 160),
    ('conv_offset_mask_small', 256, 216, 40), ('conv_offset_mask_medium', 128, 216, 80),
    ('conv_offset_mask_large', 64, 216, 160),
    ('tail_small', 64, 256, 40), ('tail_medium', 64, 256, 80), ('tail_large0', 64, 32, 160),
    ('tail_large2', 32, 3, 160), ('conv_first', 3, 64, 40),
]


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


def shape_times(cin, cout, H, iters, warmup):
    from c2m_b200 import _lib, ops
    L = _lib.lib()
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(cin * 1000 + cout)
    x = torch.randn(B, cin, H, H, device=dev, generator=g)
    w = torch.randn(cout, cin, 3, 3, device=dev, generator=g) / (3 * cin ** 0.5)
    gy = torch.randn(B, cout, H, H, device=dev, generator=g) * 2.0 ** -19
    st = torch.cuda.current_stream().cuda_stream
    xp, x_amax = ops._conv3x3_operand(x)
    gp = ops.PSA.empty(B, cout, H, H, dev)
    amax = torch.empty(B, dtype=torch.int32, device=dev)
    wt = w.transpose(0, 1)
    blob = ops.conv3x3_pack_weights(w, dgrad=True)
    nws = L.c2m_conv3x3_wgrad_workspace_bytes(B, cin, cout, H, H)
    ws = torch.empty(nws, dtype=torch.uint8, device=dev)
    dw = torch.empty_like(w)

    def convert():
        _lib.check(L.c2m_conv3x3_operand_f32(gy.data_ptr(), B, cout, H, H, *gy.stride(), gp.hi.data_ptr(),
                                             gp.lo.data_ptr(), amax.data_ptr(), st), 'grad_psa')

    def tc_dx():
        convert()
        ops.conv3x3_psa(gp, wt, None, psa_out=False, out_f32=True, packed=blob, x_amax=amax)

    def tc_dw():
        _lib.check(L.c2m_conv3x3_wgrad_scaled(gp.hi.data_ptr(), gp.lo.data_ptr(), amax.data_ptr(), xp.hi.data_ptr(),
                                       xp.lo.data_ptr(), x_amax.data_ptr(), B, cin, cout, H, H, dw.data_ptr(), ws.data_ptr(), nws, st),
                   'wgrad')

    def cudnn_dx():
        torch.nn.grad.conv2d_input(x.shape, w, gy, 1, 1)

    def cudnn_dw():
        torch.nn.grad.conv2d_weight(x, w.shape, gy, 1, 1)

    convert()
    r = {'convert_ms': timed(convert, iters, warmup), 'tc_dx_ms': timed(tc_dx, iters, warmup),
         'tc_dw_ms': timed(tc_dw, iters, warmup)}
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        sfx = 'tf32' if tf32 else 'fp32'
        r[f'cudnn_{sfx}_dx_ms'] = timed(cudnn_dx, iters, warmup)
        r[f'cudnn_{sfx}_dw_ms'] = timed(cudnn_dw, iters, warmup)
    torch.backends.cudnn.allow_tf32 = False
    r['gflop_each'] = 2.0 * B * H * H * cin * cout * 9 / 1e9
    return r


def net_step_times(iters, warmup):
    """One RestorationNet(64, 16, 8) forward + backward (L1 loss) at the stage-3 shape on each path, ms."""
    import seeding
    from mmsr.models.archs.corres_generation_arch import CorrespondenceGenerationArch
    from mmsr.models.archs.ref_restoration_arch import RestorationNet
    dev = 'cuda:0'
    net_map = CorrespondenceGenerationArch(3, 1, ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19')
    net_map.load_state_dict(seeding.seeded_state_dict(seeding.spec_net_map(), 12))
    net_map.to(dev).eval()
    net_g = RestorationNet(64, 16, 8)
    net_g.load_state_dict(seeding.seeded_state_dict(seeding.spec_restoration_net(), 13))
    net_g.to(dev).train()
    lr = 40
    hr = seeding.structured_image(31, B, 4 * lr).to(dev)
    x = F.interpolate(hr, scale_factor=0.25, mode='bicubic', align_corners=False).clamp(0, 1)
    f1 = seeding.randn(32, (B, 256, lr, lr)).to(dev)
    f2 = (f1 + seeding.randn(33, (B, 256, lr, lr), 0.1).to(dev)).roll(3, 3)
    with torch.no_grad():
        pre, feats = net_map({'dense_features1': f1, 'dense_features2': f2}, seeding.structured_image(34, B, 4 * lr).to(dev))

    def step():
        net_g.zero_grad(set_to_none=True)
        F.l1_loss(net_g(x, pre, feats), hr).backward()

    out = {}
    for name, fast, tf32 in (('tensor_core', '1', False), ('cudnn_fp32', '0', False), ('cudnn_tf32', '0', True)):
        os.environ['C2M_FAST_CONV'] = fast
        torch.backends.cudnn.allow_tf32 = tf32
        out[f'net_g_step_{name}_ms'] = timed(step, iters, warmup)
    os.environ['C2M_FAST_CONV'] = '1'
    torch.backends.cudnn.allow_tf32 = False
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None, help='JSON file for the results (default: print only)')
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {'card': card(), 'batch': B, 'shapes': {}}
    print(res['card'])
    print(f'{"shape":26s} {"Cin":>4s} {"Cout":>4s} {"HxW":>7s} | {"conv":>6s} {"tc dX":>7s} {"fp32":>7s} {"tf32":>7s} | '
          f'{"tc dW":>7s} {"fp32":>7s} {"tf32":>7s}  (ms)')
    for name, cin, cout, H in SHAPES:
        r = shape_times(cin, cout, H, args.iters, args.warmup)
        res['shapes'][name] = dict(r, Cin=cin, Cout=cout, H=H)
        print(f'{name:26s} {cin:4d} {cout:4d} {H:>3d}x{H:<3d} | {r["convert_ms"]:6.3f} {r["tc_dx_ms"]:7.3f} '
              f'{r["cudnn_fp32_dx_ms"]:7.3f} {r["cudnn_tf32_dx_ms"]:7.3f} | {r["tc_dw_ms"]:7.3f} '
              f'{r["cudnn_fp32_dw_ms"]:7.3f} {r["cudnn_tf32_dw_ms"]:7.3f}', flush=True)
    res.update(net_step_times(max(3, args.iters // 4), 2))
    for k in ('net_g_step_tensor_core_ms', 'net_g_step_cudnn_fp32_ms', 'net_g_step_cudnn_tf32_ms'):
        print(f'{k}: {res[k]:.1f}')
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
