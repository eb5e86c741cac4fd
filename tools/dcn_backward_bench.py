"""Device time of the deformable convolution's backward at the stage-3 training shapes (batch 9, dg 8, Cout = C:
256 ch at 40x40, 128 at 80x80, 64 at 160x160; offsets from a pyramid of a random index map plus N(0, 0.5^2) residuals,
sigmoid masks):
  * `_ext.dcn_v2_backward` whole, and its pieces one by one: the gcol GEMM (fp32 torch.matmul), col2im_coord, the
    atomic col2im (with the zero fill of grad_input), im2col and the dW GEMM;
  * the tensor-core backward (ops.dcn_v2_tc): whole with and without grad_input, its input conversion (grad_output to
    PSA and the operand x_il) on its own, and its dgrad / wgrad kernels from the library's profiling hook;
  * one RestorationNet(64, 16, 8) forward + backward with C2M_DCN_TC at 1 and 0, alternated.
CUDA events, medians.  Prints the card and its power limit from the same run; --out FILE writes the numbers as JSON."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')]

SHAPES = [(256, 40), (128, 80), (64, 160)]


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def _inputs(C, S, dev, B=9, dg=8):
    import seeding
    g = torch.Generator().manual_seed(C)
    x = seeding.randn(1, (B, C, S, S)).to(dev)
    far = torch.randint(-S // 2, S // 2 + 1, (B, 1, 2, S, S), generator=g).float()
    off = (far.expand(B, dg * 9, 2, S, S) + seeding.randn(2, (B, dg * 9, 2, S, S), 0.5)).reshape(B, 18 * dg, S, S).to(dev)
    mask = torch.sigmoid(seeding.randn(3, (B, dg * 9, S, S))).to(dev)
    w = seeding.randn(4, (C, C, 3, 3), (9 * C) ** -0.5).to(dev)
    b = seeding.randn(5, (C,), 0.1).to(dev)
    gy = seeding.randn(6, (B, C, S, S), 2.0 ** -19).to(dev)
    return x, off, mask, w, b, gy


def ext_pieces(x, off, mask, w, gy, reps, dg=8):
    """The pieces of `_ext.dcn_v2_backward` (ops._deform_backward at groups = 1), each timed on its own."""
    from c2m_b200 import _lib, ops
    L = _lib.lib()
    B, C, H, W = x.shape
    P = H * W
    s = ops._shape(x, C, 3, 3, 1, 1, 1, 1, 1, 1, dg, gy)
    wg, gg = w.view(1, C, C * 9), gy.view(B, 1, C, P)
    gcol = torch.matmul(wg.transpose(1, 2), gg).contiguous()
    goff, gm, gi = torch.empty_like(off), torch.empty_like(mask), torch.zeros_like(x)
    cols = torch.empty(B, C * 9, P, device=x.device)
    st = ops._stream()

    def col2im():
        gi.zero_()
        _lib.check(L.c2m_deform_conv_col2im_f32(gcol.data_ptr(), off.data_ptr(), mask.data_ptr(), s, gi.data_ptr(), st),
                   'col2im')
    return {
        'gcol_gemm': _time(lambda: torch.matmul(wg.transpose(1, 2), gg).contiguous(), reps),
        'col2im_coord': _time(lambda: _lib.check(L.c2m_deform_conv_col2im_coord_f32(
            gcol.data_ptr(), x.data_ptr(), off.data_ptr(), mask.data_ptr(), s, goff.data_ptr(), gm.data_ptr(), st),
            'col2im_coord'), reps),
        'col2im': _time(col2im, reps),
        'im2col': _time(lambda: _lib.check(L.c2m_deform_conv_im2col_f32(x.data_ptr(), off.data_ptr(), mask.data_ptr(),
                                                                         s, cols.data_ptr(), st), 'im2col'), reps),
        'dw_gemm': _time(lambda: torch.matmul(gg, cols.view(B, 1, C * 9, P).transpose(2, 3)).sum(0), reps),
    }


def conversion(x, mask, gy, reps, dg=8):
    """The tensor-core backward's input conversion: grad_output to PSA and x (with the mask's scale) to x_il."""
    from c2m_b200 import _lib, ops
    L = _lib.lib()
    B, C, H, W = x.shape
    gp = ops.PSA.empty(B, C, H, W, x.device)
    gamax = torch.empty(B, dtype=torch.int32, device=x.device)
    x_il = torch.empty(L.c2m_dcn_tc_operand_bytes(B, C, H, W, dg) // 2, dtype=torch.float16, device=x.device)
    amax = torch.empty(2 * B, dtype=torch.int32, device=x.device)
    st = ops._stream()

    def run():
        _lib.check(L.c2m_conv3x3_operand_f32(gy.data_ptr(), B, C, H, W, *gy.stride(), gp.hi.data_ptr(),
                                             gp.lo.data_ptr(), gamax.data_ptr(), st), 'conv3x3_operand_f32')
        _lib.check(L.c2m_dcn_tc_operand_f32(x.data_ptr(), B, C, H, W, *x.stride(), dg, mask.data_ptr(),
                                            x_il.data_ptr(), amax.data_ptr(), st), 'dcn_tc_operand_f32')
    return _time(run, reps)


def layer_rows(reps):
    from c2m_b200 import ops
    dev = 'cuda'
    rows = []
    for C, S in SHAPES:
        x, off, mask, w, b, gy = _inputs(C, S, dev)
        old = _time(lambda: ops.dcn_v2_backward(x, w, b, off, mask, gy, 3, 3, 1, 1, 1, 1, 1, 1, 8), reps)
        pieces = ext_pieces(x, off, mask, w, gy, reps)
        conv = conversion(x, mask, gy, reps)
        leaves = [t.detach().clone().requires_grad_() for t in (off, mask, w, b)]

        def new(x_grad):
            xr = x.detach().clone().requires_grad_(x_grad)
            y = ops.dcn_v2_tc(xr, *leaves[:3], leaves[3], 8)
            return lambda: torch.autograd.grad(y, [xr] * x_grad + leaves, gy, retain_graph=True)
        t_gi, t_nogi = _time(new(True), reps), _time(new(False), reps)
        ops.profile_enable(True)
        ops.profile_collect('dcn_dgrad')
        ops.profile_collect('dcn_wgrad')
        new(False)()
        torch.cuda.synchronize()
        dgrad, wgrad = ops.profile_collect('dcn_dgrad')['ms'], ops.profile_collect('dcn_wgrad')['ms']
        ops.profile_enable(False)
        rows.append(dict(C=C, map=S, ext_backward_ms=old, ext_pieces_ms=pieces, tc_backward_ms=t_gi,
                         tc_backward_no_grad_input_ms=t_nogi, tc_conversion_ms=conv, tc_dgrad_ms=dgrad,
                         tc_wgrad_reduce_ms=wgrad))
        print(f'C={C:3d} {S}x{S}: _ext {old:7.3f} ms (' + ', '.join(f'{k} {v:.3f}' for k, v in pieces.items()) +
              f') | tensor cores {t_gi:7.3f} ms, without grad_input {t_nogi:7.3f} ms '
              f'(conversion {conv:.3f}, dgrad {dgrad:.3f}, wgrad + reduce {wgrad:.3f})', flush=True)
    return rows


def net_rows(reps):
    import seeding
    from mmsr.models.archs.corres_generation_arch import CorrespondenceGenerationArch
    from mmsr.models.archs.ref_restoration_arch import RestorationNet
    dev = 'cuda'
    net_map = CorrespondenceGenerationArch(3, 1, ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg19')
    net_map.load_state_dict(seeding.seeded_state_dict(seeding.spec_net_map(), 12))
    net_map.to(dev).eval()
    net_g = RestorationNet(64, 16, 8)
    net_g.load_state_dict(seeding.seeded_state_dict(seeding.spec_restoration_net(), 13))
    net_g.to(dev).train()
    B, lr = 9, 40
    hr = seeding.structured_image(31, B, 4 * lr).to(dev)
    x = F.interpolate(hr, scale_factor=0.25, mode='bicubic', align_corners=False).clamp(0, 1)
    f1 = seeding.randn(32, (B, 256, lr, lr)).to(dev)
    f2 = (f1 + seeding.randn(33, (B, 256, lr, lr), 0.1).to(dev)).roll(3, 3)
    img_ref = seeding.structured_image(34, B, 4 * lr).to(dev)
    with torch.no_grad():
        pre, feats = net_map({'dense_features1': f1, 'dense_features2': f2}, img_ref)

    def step():
        net_g.zero_grad(set_to_none=True)
        F.l1_loss(net_g(x, pre, feats), hr).backward()
    times = {'1': [], '0': []}
    for flag in ('1', '0'):
        os.environ['C2M_DCN_TC'] = flag
        step()
    for _ in range(reps):
        for flag in ('1', '0'):
            os.environ['C2M_DCN_TC'] = flag
            times[flag].append(_time(step, 1))
    os.environ.pop('C2M_DCN_TC', None)
    res = {f'C2M_DCN_TC={k}': statistics.median(v) for k, v in times.items()}
    print(f'RestorationNet(64, 16, 8) forward + backward, batch 9, LR 40: ' +
          ', '.join(f'{k} {v:.1f} ms' for k, v in res.items()), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('dcn_backward_bench: needs a CUDA device')
    import __graft_entry__ as g
    g.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f'card: {card}')
    res = dict(card=card, layers=layer_rows(a.reps), restoration_net=net_rows(a.reps))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
