"""Pixel-loss training of the restoration network through `RefRestorationModel` and `mmsr/train.py`, -m gpu:
gradients of one `optimize_parameters` step against fp64 CPU autograd through the oracle, packed weights after an
in-place Adam update, bit-identical resume, kernel routing at the stage-3 shapes, the CLI end to end (one process,
and two ranks under torchrun when two GPUs are present)."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F


pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN_FIXTURE = os.path.join(ROOT, 'tests', 'fixtures', 'train_c2m_synth.yml')
TEST_FIXTURE = os.path.join(ROOT, 'tests', 'fixtures', 'test_c2m_synth.yml')


@pytest.fixture(scope='module', autouse=True)
def _native_built():
    import __graft_entry__ as g
    g.build()


def _opt(tmp_path, **train):
    t = {'lr_g': 1e-4, 'lr_offset': 1e-4, 'lr_relu2_offset': 1e-5, 'lr_relu3_offset': 1e-6, 'weight_decay_g': 0,
         'beta_g': [0.9, 0.999], 'lr_scheme': 'MultiStepLR', 'niter': 10, 'warmup_iter': -1,
         'net_g_pretrain_steps': 0, 'lr_steps': [3], 'lr_gamma': 0.5, 'pixel_criterion': 'L1Loss',
         'pixel_weight': 1.0, 'manual_seed': 10}
    t.update(train)
    for d in ('models', 'training_state', 'visualization'):
        os.makedirs(tmp_path / d, exist_ok=True)
    return {'name': 'traintest', 'suffix': None, 'scale': 4, 'crop_border': None, 'dist': False, 'is_train': True,
            'network_g': {'type': 'RestorationNet', 'ngf': 64, 'n_blocks': 16, 'groups': 8},
            'network_map': {'type': 'CorrespondenceGenerationArch', 'patch_size': 3, 'stride': 1,
                            'vgg_layer_list': ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg_type': 'vgg19',
                            'vgg_pretrained': False},
            'network_extractor': {'type': 'ContrasExtractorSep'}, 'train': t,
            'path': {'models': str(tmp_path / 'models'), 'training_state': str(tmp_path / 'training_state'),
                     'visualization': str(tmp_path / 'visualization'), 'strict_load': True}}


def _model(opt, weights=True):
    import copy
    import bench
    from mmsr.models.ref_restoration_model import RefRestorationModel, _bare
    model = RefRestorationModel(copy.deepcopy(opt))
    if weights:
        for net, sd in zip((model.net_extractor, model.net_map, _bare(model.net_g)), bench.seeded_weights()):
            net.load_state_dict(sd, strict=True)
    return model


def _batches(n, batch, gt, seed=0):
    import random
    from mmsr.data import create_dataset
    ds = create_dataset({'name': 's', 'type': 'SyntheticRefDataset', 'phase': 'train', 'scale': 4, 'num': n * batch,
                         'gt_size': gt, 'in_size': gt + 16, 'ref_size': gt + 20, 'use_flip': True, 'use_rot': True})
    random.seed(seed)
    out = []
    for b in range(n):
        samples = [ds[b * batch + k] for k in range(batch)]
        out.append({k: torch.stack([s[k] for s in samples]) for k in samples[0]})
    return out


def test_step_gradients_match_fp64_oracle(tmp_path):
    """One optimize_parameters step (B = 2, LR 40x40): every net_g gradient against fp64 CPU autograd of the same L1
    loss through oracle.ref_path.restoration_net on the same inputs, pre-offsets and Ref features, as the largest
    absolute error over the gradient's largest magnitude.  Bar: 1e-4 for the layers after the last deformable
    convolution (head_large, body_large, tail_large), 1e-3 for every parameter.  The gradient of a bilinear sample
    with respect to its offset jumps where the sample crosses a pixel boundary, so the rounding-level difference
    between the fp32 and the fp64 forward moves a few samples across one and changes the gradients of everything
    upstream of the offsets by more than the kernels' own error (measured on an H100: 6.7e-4 at
    small_dyn_agg.conv_offset_mask.weight, 7.5e-5 after the last DCN at body_large.12.conv1.weight, no L1 sign
    flips)."""
    from oracle import ref_path
    model = _model(_opt(tmp_path))
    sd0 = {k: v.detach().cpu().double() for k, v in model.net_g.state_dict().items()}
    model.feed_data(_batches(1, 2, 160)[0])
    model.update_learning_rate(1)
    model.optimize_parameters(1)
    torch.cuda.synchronize()
    got = {n: p.grad.detach().cpu().double() for n, p in model.net_g.named_parameters()}
    pre = {k: model.pre_offset[k].cpu().double() for k in ('relu1_1', 'relu2_1', 'relu3_1')}
    feats = {k: model.img_ref_feat[k].cpu().double() for k in ('relu1_1', 'relu2_1', 'relu3_1')}
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd0.items()}
    torch.set_num_threads(os.cpu_count() or 1)
    out = ref_path.restoration_net(leaves, model.img_in_lq.cpu().double(), pre, feats)
    gt = model.gt.cpu().double()
    F.l1_loss(out, gt).backward()
    flips = int(((out.detach() - gt).sign() != (model.output.detach().cpu().double() - gt).sign()).sum())
    ratio = {n: float((got[n] - leaves[n].grad).abs().max() / leaves[n].grad.abs().max().clamp_min(1e-300))
             for n in got}
    after = {n: r for n, r in ratio.items() if n.split('.')[1] in ('head_large', 'body_large', 'tail_large')}
    worst, worst_after = max(ratio.items(), key=lambda kv: kv[1]), max(after.items(), key=lambda kv: kv[1])
    print(f'worst gradient error / largest magnitude {worst[1]:.3e} at {worst[0]}; after the last DCN '
          f'{worst_after[1]:.3e} at {worst_after[0]}; L1 sign flips {flips}')
    assert len(after) == 2 + 2 * 2 * 16 + 4 and flips == 0
    assert worst_after[1] <= 1e-4, worst_after
    assert worst[1] <= 1e-3, worst


def test_packed_weights_refresh_after_a_step(tmp_path):
    """Adam updates net_g in place; the packed-weight caches key on the tensor version, so a forward after the step
    equals, bit for bit, the forward of a fresh RestorationNet loaded with the updated state dict."""
    from mmsr.models.archs.ref_restoration_arch import RestorationNet
    model = _model(_opt(tmp_path))
    model.feed_data(_batches(1, 2, 160)[0])
    model.test()                                  # fills the inference path's weight packs
    before = model.output.clone()
    model.update_learning_rate(1)
    model.optimize_parameters(1)
    model.test()
    fresh = RestorationNet(64, 16, 8)
    fresh.load_state_dict({k: v.detach().cpu() for k, v in model.net_g.state_dict().items()})
    fresh.to(DEV).eval()
    with torch.no_grad():
        want = fresh(model.img_in_lq, model.pre_offset, model.img_ref_feat)
    assert not torch.equal(model.output, before)
    assert torch.equal(model.output, want)


def _state(model):
    opt = model.optimizer_g.state_dict()
    return ({k: v.detach().clone() for k, v in model.net_g.state_dict().items()},
            {i: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in s.items()} for i, s in opt['state'].items()},
            [g['lr'] for g in opt['param_groups']])


def test_resume_is_bit_identical(tmp_path):
    """Deterministic algorithms on: 4 iterations straight equal 2 iterations, save, a rebuilt model resumed from the
    checkpoint and training state, and 2 more: net_g weights, Adam state and learning rates bit for bit."""
    batches = _batches(4, 2, 96)
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        def run(model, iters):
            for it in iters:
                model.update_learning_rate(it)
                model.feed_data(batches[it - 1])
                model.optimize_parameters(it)
        a = _model(_opt(tmp_path / 'a'))
        run(a, range(1, 5))
        b = _model(_opt(tmp_path / 'b'))
        run(b, range(1, 3))
        b.save(0, 2)
        opt_c = _opt(tmp_path / 'b')
        opt_c['path']['pretrain_model_g'] = str(tmp_path / 'b' / 'models' / 'net_g_2.pth')
        c = _model(opt_c, weights=False)
        import bench
        sd_e, sd_m, _ = bench.seeded_weights()
        c.net_extractor.load_state_dict(sd_e)
        c.net_map.load_state_dict(sd_m)
        c.resume_training(torch.load(tmp_path / 'b' / 'training_state' / '2.state', weights_only=False))
        run(c, range(3, 5))
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    wa, sa, la = _state(a)
    wc, sc, lc = _state(c)
    assert la == lc and la[0] == 0.5e-4           # lr_steps [3]: halved from iteration 4 on
    assert wa.keys() == wc.keys() and all(torch.equal(wa[k], wc[k]) for k in wa)
    assert sa.keys() == sc.keys()
    for i in sa:
        for k in sa[i]:
            assert (torch.equal(sa[i][k], sc[i][k]) if torch.is_tensor(sa[i][k]) else sa[i][k] == sc[i][k]), (i, k)
    ckpt = torch.load(tmp_path / 'b' / 'models' / 'net_g_2.pth')
    assert not any(k.startswith('module.') for k in ckpt)


def test_stage3_step_runs_on_the_library_kernels(tmp_path, monkeypatch):
    """A training step at the stage-3 shapes (batch 9, GT 160: LR 40x40, Ref 160x160): every convolution of net_g
    runs forward / dX on the 3x3 kernel and dW on its weight-gradient kernel, every DCN forward on the tensor-core
    DCN and its backward on dgrad / wgrad; no cuDNN convolution inside net_g and no `_ext` backward."""
    import _ext
    from c2m_b200 import _lib, ops
    model = _model(_opt(tmp_path))
    model.feed_data(_batches(1, 9, 160)[0])
    model.update_learning_rate(1)
    model.optimize_parameters(1)                   # warm-up: packs, workspaces
    torch.cuda.synchronize()
    L = _lib.lib()
    calls = []
    for name in ('c2m_deform_conv_col2im_coord_f32', 'c2m_deform_conv_im2col_f32', 'c2m_deform_conv_col2im_f32',
                 'c2m_deform_conv_col2im_det_f32'):
        fn = getattr(L, name)
        monkeypatch.setattr(L, name, lambda *a, _fn=fn, _n=name: calls.append(_n) or _fn(*a), raising=False)
    for name in ('dcn_v2_backward', 'dcn_v2_forward'):
        fn = getattr(_ext, name)
        monkeypatch.setattr(_ext, name, lambda *a, _fn=fn, _n=name: calls.append(_n) or _fn(*a))
    inside, cudnn = [False], {'net_g': 0, 'other': 0}
    conv2d = F.conv2d

    def spy(*a, **k):
        cudnn['net_g' if inside[0] else 'other'] += 1
        return conv2d(*a, **k)
    monkeypatch.setattr(F, 'conv2d', spy)
    h1 = model.net_g.register_forward_pre_hook(lambda *a: inside.__setitem__(0, True))
    h2 = model.net_g.register_forward_hook(lambda *a: inside.__setitem__(0, False))
    kinds = ('conv3x3', 'conv3x3_wgrad', 'dcn', 'dcn_dgrad', 'dcn_wgrad')
    ops.profile_enable(True)
    for k in kinds:
        ops.profile_collect(k)
    try:
        model.update_learning_rate(2)
        model.optimize_parameters(2)
        torch.cuda.synchronize()
        n = {k: ops.profile_collect(k)['launches'] for k in kinds}
    finally:
        ops.profile_enable(False)
        h1.remove()
        h2.remove()
        monkeypatch.undo()
    n_conv = sum(isinstance(m, torch.nn.Conv2d) for m in model.net_g.modules())
    print(f'launches {n}; {n_conv} convolutions in net_g; F.conv2d calls {cudnn}; _ext / CUDA-core DCN calls {calls}')
    assert cudnn['net_g'] == 0 and not calls, (cudnn, calls)
    assert n['conv3x3_wgrad'] >= n_conv and n['conv3x3'] >= n_conv, (n, n_conv)
    assert n['dcn_dgrad'] == 3 and n['dcn_wgrad'] == 3, n
    assert torch.isfinite(torch.tensor(model.get_current_log()['l_g_pix']))


def _train_yaml(tmp_path, exp, **extra):
    text = open(TRAIN_FIXTURE).read().replace('  resume_state: ~', f'  resume_state: ~\n  experiments_root: {exp}')
    for k, v in extra.items():
        text = text.replace(k, v)
    p = tmp_path / 'train.yml'
    p.write_text(text)
    return str(p)


def _run(cmd, **kw):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, 'c2-matching_b200'),
                                                       os.environ.get('PYTHONPATH', '')]))
    return subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, **kw)


def test_train_cli_end_to_end(tmp_path):
    """`mmsr/train.py -opt tests/fixtures/train_c2m_synth.yml` (run directory moved to a temporary one): exits 0,
    writes net_g checkpoints and training states, logs finite losses, validates; test.py loads the checkpoint strictly."""
    import math
    import re
    exp = tmp_path / 'exp'
    r = _run([sys.executable, os.path.join(ROOT, 'c2-matching_b200', 'mmsr', 'train.py'), '-opt',
              _train_yaml(tmp_path, exp)])
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    for f in ('models/net_g_2.pth', 'models/net_g_4.pth', 'models/net_g_latest.pth', 'training_state/2.state',
              'training_state/4.state'):
        assert (exp / f).is_file(), f
    losses = [float(v) for v in re.findall(r'l_g_pix: (\S+)', out)]
    assert len(losses) == 4 and all(math.isfinite(v) for v in losses), losses
    assert out.count('# Validation synth_val # PSNR:') == 2
    lr = re.findall(r'lr:\((\S+?),', out)
    assert [float(v) for v in lr] == [1e-4, 1e-4, 1e-4, 1e-5], lr          # lr_steps [3], lr_gamma 0.1
    state = torch.load(exp / 'training_state' / '4.state', weights_only=False)
    assert state['iter'] == 4 and len(state['optimizers']) == 1 and len(state['schedulers']) == 1
    text = open(TEST_FIXTURE).read().replace('name: c2m_synth', 'name: c2m_synth_trained').replace(
        '  pretrain_model_g: ~', f"  pretrain_model_g: {exp / 'models' / 'net_g_latest.pth'}")
    (tmp_path / 'test.yml').write_text(text)
    r = _run([sys.executable, os.path.join(ROOT, 'c2-matching_b200', 'mmsr', 'test.py'), '-opt',
              str(tmp_path / 'test.yml')])
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert 'Loading RestorationNet model from' in r.stdout + r.stderr
    assert '# Validation synth # PSNR:' in r.stdout + r.stderr


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_train_cli_two_ranks_keep_equal_weights(tmp_path):
    """torchrun with two ranks on the same fixture (batch 2 = 1 per rank): after the run every rank holds the same
    net_g weights."""
    exp = tmp_path / 'exp'
    script = tmp_path / 'run_ranks.py'
    script.write_text(
        'import sys, torch\n'
        f"sys.path[:0] = [{os.path.join(ROOT, 'c2-matching_b200')!r}]\n"
        'import mmsr.models.ref_restoration_model as m\n'
        'orig = m.RefRestorationModel.save\n'
        'def save(self, epoch, it):\n'
        '    if it == -1:\n'
        f"        torch.save(m._bare(self.net_g).state_dict(), {str(tmp_path)!r} + f'/rank{{torch.distributed.get_rank()}}.pth')\n"
        '    return orig(self, epoch, it)\n'
        'm.RefRestorationModel.save = save\n'
        'from mmsr import train\n'
        'train.main()\n')
    r = _run([sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc_per_node', '2', str(script),
              '-opt', _train_yaml(tmp_path, exp), '--launcher', 'pytorch'])
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    a, b = torch.load(tmp_path / 'rank0.pth'), torch.load(tmp_path / 'rank1.pth')
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert (exp / 'models' / 'net_g_latest.pth').is_file()
