"""Test infrastructure (kept under tests/ because it calls the oracle): diagnostic run on the GPU box,
every kernel vs the oracle, mismatch statistics printed (no
asserts) so one gpurun call tells as much as possible.  Not a test, not a benchmark."""
import os
import sys
import time
import traceback

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')):
    sys.path.insert(0, p)
import make_golden as mg  # noqa: E402
import seeding  # noqa: E402
from oracle import c_oracle, ref_path  # noqa: E402
import c2m_b200 as c2m  # noqa: E402

dev = torch.device('cuda:0')
G = {n: np.load(os.path.join(ROOT, 'tests', 'golden', n + '.npz')) for n in ('corr', 'offsets', 'dcn', 'full')}


def section(name):
    print(f'\n===== {name} =====', flush=True)


def corr_diag():
    section('corr vs golden')
    for case in mg.CORR_CASES:
        name = case[0]
        fin, fref = mg.corr_inputs(case)
        ref_idx = G['corr'][f'{name}/ni1/idx']
        ref_val = G['corr'][f'{name}/ni1/val']
        for force in (True, False):
            try:
                idx, val = c2m.corr_argmax(fin[None].to(dev), fref[None].to(dev), is_norm=True, norm_input=True,
                                           force_generic=force)
                torch.cuda.synchronize()
                idx = idx[0].cpu().numpy()
                val = val[0].cpu().numpy()
                bad = int((idx != ref_idx).sum())
                dv = float(np.abs(val - ref_val).max())
                print(f'{name:14s} generic={force!s:5s} idx mismatches {bad}/{idx.size}  max|dval| {dv:.3e}', flush=True)
                if bad and bad < 20:
                    ys, xs = np.nonzero(idx != ref_idx)
                    for y, x in list(zip(ys, xs))[:5]:
                        print(f'    q=({y},{x}) got {idx[y, x]} want {ref_idx[y, x]} val {val[y, x]:.6f} vs {ref_val[y, x]:.6f}')
            except Exception:
                traceback.print_exc()


def corr_big():
    section('corr big (160x160 maps, 256ch) umma vs generic, timing')
    for (B, h, hr) in ((1, 40, 125), (1, 160, 160), (4, 160, 160)):
        fin = torch.stack([seeding.unit_features(900 + b, 256, h, h) for b in range(B)]).to(dev)
        fref = torch.stack([seeding.unit_features(950 + b, 256, hr, hr) for b in range(B)]).to(dev)
        res = {}
        for force in (False, True):
            if force and B > 1:
                continue
            try:
                for it in range(3):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    idx, val = c2m.corr_argmax(fin, fref, is_norm=True, norm_input=True, force_generic=force)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                res[force] = (idx.cpu(), val.cpu())
                nq = idx[0].numel()
                nr = (hr - 2) ** 2
                fl = 2 * 2304 * nq * nr * B
                print(f'B={B} {h}x{h} vs {hr}x{hr} generic={force}: {dt * 1e3:.2f} ms  ({fl / dt / 1e12:.1f} TFLOP/s algorithmic)', flush=True)
            except Exception:
                traceback.print_exc()
        if True in res and False in res:
            bad = int((res[True][0] != res[False][0]).sum())
            print(f'   umma vs generic idx mismatches: {bad}; max|dval| {float((res[True][1] - res[False][1]).abs().max()):.3e}')
        if h <= 40 and False in res:
            t0 = time.perf_counter()
            oi, ov = ref_path.feature_match_index(fin[0].cpu(), fref[0].cpu(), 3, 1, 1, True, True)
            print(f'   torch-cpu oracle {time.perf_counter() - t0:.2f}s; idx mismatches vs oracle: {int((oi != res[False][0][0]).sum())}')


def offsets_diag():
    section('offset pyramid')
    idx = torch.randint(0, 12 * 14, (2, 12, 14), dtype=torch.int64)
    for s in (1, 2, 4):
        got = c2m.offset_pyramid(idx.to(dev), s).cpu()
        want = torch.stack([c_oracle.offset_pyramid(idx[b], s) for b in range(2)])
        print(f'scale {s}: equal={torch.equal(got, want)}')


def dcn_diag():
    section('dcn vs literal C oracle / golden')
    import _ext
    for case in mg.DCN_CASES:
        name, b, c, cout, h, w, dg, seed, osc = case
        x = seeding.randn(seed, (b, c, h, w))
        wgt = seeding.randn(seed + 5, (cout, c, 3, 3), 0.1)
        bias = seeding.randn(seed + 6, (cout,))
        off = seeding.randn(seed + 7, (b, 2 * dg * 9, h, w), 2.0 * osc)
        off[:, :, ::2, ::3] = off[:, :, ::2, ::3].round()
        mask = torch.sigmoid(seeding.randn(seed + 8, (b, dg * 9, h, w)))
        want = c_oracle.dcn_v2_forward(x, wgt, bias, off, mask, dg=dg, acc64=True)
        try:
            got = _ext.dcn_v2_forward(x.to(dev), wgt.to(dev), bias.to(dev), off.to(dev), mask.to(dev), 3, 3, 1, 1, 1, 1, 1, 1, dg).cpu()
            print(f'{name}: _ext max abs err {float((got - want).abs().max()):.3e} (out rms {float(want.pow(2).mean().sqrt()):.3f})')
            got = _ext.dcn_v2_forward(x.to(dev).contiguous(memory_format=torch.channels_last), wgt.to(dev), bias.to(dev), off.to(dev), mask.to(dev), 3, 3, 1, 1, 1, 1, 1, 1, dg).cpu()
            print(f'{name}: _ext(channels_last x) max abs err {float((got - want).abs().max()):.3e}')
        except Exception:
            traceback.print_exc()
    # timing at BASELINE config 4 and the three full-size layers
    section('dcn timing')
    for (C, H, B) in ((64, 160, 1), (256, 160, 1), (128, 320, 1), (64, 640, 1)):
        x = torch.randn(B, C, H, H, device=dev)
        wgt = torch.randn(C, C, 3, 3, device=dev) * 0.05
        bias = torch.randn(C, device=dev)
        off = torch.randn(B, 144, H, H, device=dev) * 3
        mask = torch.sigmoid(torch.randn(B, 72, H, H, device=dev))
        import torchvision
        for tag, fn in (('c2m', lambda: _ext.dcn_v2_forward(x, wgt, bias, off, mask, 3, 3, 1, 1, 1, 1, 1, 1, 8)),
                        ('c2m-nhwc', lambda: _ext.dcn_v2_forward(x.contiguous(memory_format=torch.channels_last), wgt, bias, off, mask, 3, 3, 1, 1, 1, 1, 1, 1, 8)),
                        ('torchvision', lambda: torchvision.ops.deform_conv2d(x, off, wgt, bias, padding=1, mask=mask))):
            try:
                for _ in range(2):
                    y = fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(5):
                    y = fn()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / 5
                print(f'C={C} H={H}: {tag:12s} {ms:.3f} ms  ({2 * C * C * 9 * H * H / ms / 1e9:.1f} TFLOP/s)', flush=True)
            except Exception:
                traceback.print_exc()


def conv_diag():
    section('conv3x3 tensor-core (fp16x3) vs fp64 reference')
    import torch.nn.functional as F
    from c2m_b200 import ops
    for (B, cin, cout, H, W, act, res) in ((2, 64, 64, 40, 44, 'relu', False), (1, 64, 64, 37, 29, None, True),
                                           (1, 64, 32, 32, 32, 'lrelu', False), (1, 32, 3, 48, 40, None, False),
                                           (2, 3, 64, 32, 24, 'lrelu', False), (1, 24, 40, 33, 21, 'relu', True)):
        try:
            x = seeding.randn(1, (B, cin, H, W), 1.5)
            w = seeding.randn(2, (cout, cin, 3, 3), 0.05)
            b = seeding.randn(3, (cout,), 0.5)
            r = seeding.randn(4, (B, cout, H, W)) if res else None
            want = F.conv2d(x.double(), w.double(), b.double(), 1, 1)
            if act == 'relu':
                want = want.relu()
            elif act == 'lrelu':
                want = F.leaky_relu(want, 0.1)
            if res:
                want = want + r.double()
            xp = ops.psa_from_f32(x.to(dev))
            back = ops.psa_to_f32(xp).cpu()
            rp = ops.psa_from_f32(r.to(dev)) if res else None
            yp = ops.conv3x3_psa(xp, w.to(dev), b.to(dev), act=act, residual=rp)
            got = ops.psa_to_f32(yp).cpu()
            torch.cuda.synchronize()
            torch.backends.cudnn.allow_tf32 = False
            cud = F.conv2d(x.to(dev), w.to(dev), b.to(dev), 1, 1).cpu()
            print(f'B{B} {cin}->{cout} {H}x{W} act={act} res={res}: psa roundtrip err {float((back - x).abs().max()):.2e}; '
                  f'conv max err {float((got.double() - want).abs().max()):.3e} (scale {float(want.abs().max()):.2f}); '
                  f'[cuDNN fp32 pre-act err {float((cud.double() - F.conv2d(x.double(), w.double(), b.double(), 1, 1)).abs().max()):.3e}]', flush=True)
        except Exception:
            traceback.print_exc()
    section('conv3x3 general: dual input / slices / pixel shuffle / fp32 out')
    for (B, c1, c2, cout, H, W, act, mode) in ((1, 64, 256, 256, 40, 40, 'lrelu', 'psa'), (2, 64, 128, 128, 24, 40, 'lrelu', 'psa'),
                                               (1, 128, 0, 216, 36, 30, None, 'f32'), (1, 64, 0, 256, 32, 24, 'lrelu', 'ps2'),
                                               (1, 256, 0, 256, 20, 26, 'relu', 'both'), (1, 32, 0, 3, 40, 48, None, 'f32add'),
                                               (1, 64, 64, 64, 130, 70, 'lrelu', 'psa')):
        try:
            x1 = seeding.randn(11, (B, c1, H, W), 1.2)
            x2 = seeding.randn(12, (B, c2, H, W), 0.8) if c2 else None
            cin = c1 + c2
            w = seeding.randn(13, (cout, cin, 3, 3), 0.03)
            b = seeding.randn(14, (cout,), 0.5)
            xin = torch.cat([x1, x2], 1) if c2 else x1
            want = F.conv2d(xin.double(), w.double(), b.double(), 1, 1)
            want = want.relu() if act == 'relu' else F.leaky_relu(want, 0.1) if act == 'lrelu' else want
            p1 = ops.psa_from_f32(x1.to(dev))
            p2 = ops.psa_from_f32(x2.to(dev)) if c2 else None
            wd, bd = w.to(dev), b.to(dev)
            if mode == 'psa':
                got = ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2)).cpu()
            elif mode == 'f32':
                got = ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, psa_out=False, out_f32=True).cpu()
            elif mode == 'f32add':
                add = seeding.randn(15, (B, cout, H, W))
                got = ops.conv3x3_psa(p1, wd, bd, act=act, x2=p2, psa_out=False, out_f32=True, add_f32=add.to(dev)).cpu()
                want = want + add.double()
            elif mode == 'ps2':
                got = ops.psa_to_f32(ops.conv3x3_psa(p1, wd, bd, act=act, pixel_shuffle=2)).cpu()
                want = F.pixel_shuffle(want, 2)
            else:
                gp, gf = ops.conv3x3_psa(p1, wd, bd, act=act, out_f32=True)
                got = gf.cpu()
                print('   both: psa vs f32 diff', float((ops.psa_to_f32(gp).cpu() - got).abs().max()))
            torch.cuda.synchronize()
            print(f'B{B} {c1}+{c2}->{cout} {H}x{W} {mode}: max err {float((got.double() - want).abs().max()):.3e} (scale {float(want.abs().max()):.2f})', flush=True)
        except Exception:
            traceback.print_exc()
    section('conv3x3 timing (B=4)')
    for (cin, cout, H) in ((128, 64, 640), (64, 216, 640), (192, 128, 320), (320, 256, 160), (256, 256, 160), (64, 256, 320)):
        try:
            x = torch.randn(4, cin, H, H, device=dev)
            w = torch.randn(cout, cin, 3, 3, device=dev) * 0.03
            b = torch.randn(cout, device=dev)
            xp = ops.psa_from_f32(x)
            yp = ops.PSA.empty(4, cout, H, H, dev)
            for _ in range(3):
                ops.conv3x3_psa(xp, w, b, act='lrelu', out=yp)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                ops.conv3x3_psa(xp, w, b, act='lrelu', out=yp)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            torch.backends.cudnn.allow_tf32 = False
            for _ in range(2):
                F.conv2d(x, w, b, 1, 1)
            e0.record()
            for _ in range(3):
                F.conv2d(x, w, b, 1, 1)
            e1.record()
            torch.cuda.synchronize()
            ms_c = e0.elapsed_time(e1) / 3
            fl = 2 * cin * cout * 9 * H * H * 4
            print(f'{cin}->{cout} @{H}: c2m {ms:.3f} ms ({fl / ms / 1e9:.0f} TFLOP/s alg); cuDNN fp32 {ms_c:.3f} ms', flush=True)
        except Exception:
            traceback.print_exc()
    section('conv3x3 timing, 64->64, B=4')
    for H in (160, 320, 640):
        x = torch.randn(4, 64, H, H, device=dev)
        w = torch.randn(64, 64, 3, 3, device=dev) * 0.05
        b = torch.randn(64, device=dev)
        xp = ops.psa_from_f32(x)
        yp = ops.PSA.empty(4, 64, H, H, dev)

        def t(fn, n=10):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n
        try:
            ms = t(lambda: ops.conv3x3_psa(xp, w, b, act='relu', out=yp))
            ms_r = t(lambda: ops.conv3x3_psa(xp, w, b, act=None, residual=xp, out=yp))
            torch.backends.cudnn.allow_tf32 = False
            ms_c = t(lambda: F.conv2d(x, w, b, 1, 1), 5)
            torch.backends.cudnn.allow_tf32 = True
            ms_t = t(lambda: F.conv2d(x, w, b, 1, 1), 5)
            torch.backends.cudnn.allow_tf32 = False
            ms_cv = t(lambda: ops.psa_from_f32(x))
            fl = 2 * 64 * 64 * 9 * H * H * 4
            print(f'H={H}: c2m {ms:.3f} ms ({fl / ms / 1e9:.0f} TFLOP/s alg), +residual {ms_r:.3f} ms; cuDNN fp32 {ms_c:.3f} ms; cuDNN tf32 {ms_t:.3f} ms; psa_from_f32 {ms_cv:.3f} ms', flush=True)
        except Exception:
            traceback.print_exc()


def dcntc_diag():
    section('DCN tensor-core vs FFMA kernel / oracle')
    from c2m_b200 import ops
    for (B, C, cout, dg, gh, gw, sc) in ((1, 64, 64, 8, 10, 12, 2), (2, 16, 16, 2, 20, 9, 1), (1, 128, 128, 8, 9, 9, 2), (1, 256, 256, 8, 20, 20, 1), (1, 32, 48, 4, 18, 11, 1)):
        try:
            H, W = sc * (gh + 2), sc * (gw + 2)
            idx = torch.from_numpy(np.random.default_rng(5).integers(0, gh * gw, (B, gh, gw))).to(dev)
            x = seeding.randn(61, (B, C, H, W)).to(dev)
            om = seeding.randn(62, (B, 27 * dg, H, W), 0.7).to(dev)
            wgt = seeding.randn(63, (cout, C, 3, 3), 0.1).to(dev)
            bias = seeding.randn(64, (cout,)).to(dev)
            want = c2m.dcn_v2_fused_forward(x, om, wgt, bias, dg, idx=idx, pre_scale=sc, lrelu_slope=0.1)
            gp, gf = ops.dcn_v2_fused_tc(x, om, wgt, bias, dg, idx=idx, pre_scale=sc, lrelu=True, psa_out=True, out_f32=True)
            torch.cuda.synchronize()
            print(f'B{B} C{C}->{cout} dg{dg} {H}x{W}: tc vs ffma max diff {float((gf - want).abs().max()):.3e} (scale {float(want.abs().max()):.2f}); psa vs f32 {float((ops.psa_to_f32(gp) - gf).abs().max()):.2e}', flush=True)
            # vs the literal C oracle (fp64 accumulation)
            pre = c2m.offset_pyramid(idx, sc)
            n = dg * 9
            off = om[:, :2 * n].clone()
            pr = pre.repeat(1, dg, 1, 1, 1)
            off[:, 0::2] += pr[..., 1]
            off[:, 1::2] += pr[..., 0]
            lit = c_oracle.dcn_v2_forward(x.cpu(), wgt.cpu(), bias.cpu(), off.cpu(), torch.sigmoid(om[:, 2 * n:]).cpu(), dg=dg, acc64=True)
            lit = torch.nn.functional.leaky_relu(lit, 0.1)
            print(f'     tc vs literal oracle {float((gf.cpu() - lit).abs().max()):.3e}; ffma vs oracle {float((want.cpu() - lit).abs().max()):.3e}', flush=True)
        except Exception:
            traceback.print_exc()
    section('DCN timing B=4 (tc vs ffma)')
    for (C, H) in ((256, 160), (128, 320), (64, 640)):
        try:
            B = 4
            gh = gw = 158
            sc = H // 160
            idx = torch.randint(0, gh * gw, (B, gh, gw), device=dev)
            x = torch.randn(B, C, H, H, device=dev).contiguous(memory_format=torch.channels_last)
            xpsa = ops.psa_from_f32(x)
            om = torch.randn(B, 216, H, H, device=dev)
            wgt = torch.randn(C, C, 3, 3, device=dev) * 0.05
            bias = torch.randn(C, device=dev)

            def t(fn, n=5):
                for _ in range(2):
                    fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(n):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / n
            ms_tc = t(lambda: ops.dcn_v2_fused_tc(xpsa, om, wgt, bias, 8, idx=idx, pre_scale=sc, lrelu=True, psa_out=True, out_f32=False))
            ms_ff = t(lambda: c2m.dcn_v2_fused_forward(x, om, wgt, bias, 8, idx=idx, pre_scale=sc, lrelu_slope=0.1), 3)
            print(f'C={C} H={H}: tc {ms_tc:.3f} ms, ffma {ms_ff:.3f} ms', flush=True)
        except Exception:
            traceback.print_exc()


if __name__ == '__main__':
    print(torch.cuda.get_device_name(0), torch.__version__)
    c_oracle.build()
    which = sys.argv[1:] or ['corr', 'big', 'offsets', 'dcn']
    if 'conv' in which:
        conv_diag()
    if 'dcntc' in which:
        dcntc_diag()
    if 'corr' in which:
        corr_diag()
    if 'offsets' in which:
        offsets_diag()
    if 'dcn' in which:
        dcn_diag()
    if 'big' in which:
        corr_big()
