"""Host side of pixel-loss training of the restoration network (no GPU): options, the optimizer's parameter groups,
the learning-rate schedule, train-phase samples and augmentation, the training sampler and loader, and the options
that are out of scope."""
import collections
import os
import random

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, 'tests', 'fixtures', 'train_c2m_synth.yml')


def _train_opt(**kw):
    t = {'lr_g': 1e-4, 'lr_offset': 2e-4, 'lr_relu2_offset': 1e-5, 'lr_relu3_offset': 1e-6, 'weight_decay_g': 0,
         'beta_g': [0.9, 0.999], 'lr_scheme': 'MultiStepLR', 'lr_steps': [3, 5], 'lr_gamma': 0.1}
    t.update(kw)
    return t


def test_parse_train_fixture_gives_experiment_paths(tmp_path):
    from mmsr.utils.options import parse
    opt = parse(FIXTURE, is_train=True)
    exp = os.path.join(ROOT, 'c2-matching_b200', 'experiments', 'train_c2m_synth')
    assert opt['is_train'] is True and opt['crop_border'] == 4
    assert opt['path']['experiments_root'] == exp and opt['path']['log'] == exp
    assert opt['path']['models'] == os.path.join(exp, 'models')
    assert opt['path']['training_state'] == os.path.join(exp, 'training_state')
    assert opt['path']['visualization'] == os.path.join(exp, 'visualization')
    assert opt['datasets']['train']['phase'] == 'train' and opt['datasets']['val']['phase'] == 'val'
    assert opt['datasets']['train']['scale'] == 4
    # a run directory named in the file replaces the one under the package
    text = open(FIXTURE).read().replace('  resume_state: ~', f'  resume_state: ~\n  experiments_root: {tmp_path}')
    (tmp_path / 'o.yml').write_text(text)
    opt = parse(str(tmp_path / 'o.yml'), is_train=True)
    assert opt['path']['models'] == os.path.join(str(tmp_path), 'models')


def test_param_groups_partition_restoration_net_by_the_reference_rule():
    from mmsr.models.archs.ref_restoration_arch import RestorationNet
    from mmsr.models.ref_restoration_model import build_optimizer, param_groups
    net = RestorationNet(64, 16, 8)
    groups = param_groups(net)
    assert list(groups) == ['g', 'offset', 'relu3_offset', 'relu2_offset']
    named = dict(net.named_parameters())
    seen = [n for ps in groups.values() for n, _ in ps]
    assert sorted(seen) == sorted(named) and len(seen) == len(set(seen))
    for group, ps in groups.items():
        for n, p in ps:
            assert p is named[n]
            want = ('g' if 'offset' not in n else 'relu3_offset' if 'small' in n else
                    'relu2_offset' if 'medium' in n else 'offset')
            assert group == want, (n, group)
    by_name = {n: g for g, ps in groups.items() for n, _ in ps}
    assert by_name['dyn_agg_restore.small_offset_conv1.weight'] == 'relu3_offset'
    assert by_name['dyn_agg_restore.small_dyn_agg.conv_offset_mask.bias'] == 'relu3_offset'
    assert by_name['dyn_agg_restore.medium_offset_conv2.weight'] == 'relu2_offset'
    assert by_name['dyn_agg_restore.large_dyn_agg.conv_offset_mask.weight'] == 'offset'
    assert by_name['dyn_agg_restore.small_dyn_agg.weight'] == 'g'
    assert by_name['content_extractor.conv_first.weight'] == 'g'
    assert all(len(ps) for ps in groups.values())
    opt = build_optimizer(net, _train_opt(weight_decay_g=1e-3, beta_g=[0.5, 0.9]))
    assert [g['lr'] for g in opt.param_groups] == [1e-4, 2e-4, 1e-6, 1e-5]
    assert all(g['weight_decay'] == 1e-3 and g['betas'] == (0.5, 0.9) for g in opt.param_groups)
    assert [len(g['params']) for g in opt.param_groups] == [len(ps) for ps in groups.values()]


def _lr_trace(train_opt, iters):
    from mmsr.models.ref_restoration_model import build_scheduler, update_learning_rate
    params = [torch.nn.Parameter(torch.zeros(1)) for _ in range(2)]
    opt = torch.optim.Adam([{'params': [params[0]]}, {'params': [params[1]], 'lr': 2e-4}], lr=1e-4)
    sched = build_scheduler(opt, train_opt)
    trace = []
    for it in range(1, iters + 1):
        update_learning_rate([opt], [sched], it, train_opt.get('warmup_iter', -1))
        trace.append([g['lr'] for g in opt.param_groups])
        opt.step()
    return trace


def test_multistep_schedule_around_lr_steps():
    """The schedulers step from the second iteration on, so the lr of iteration `it` has seen the milestones
    below `it`: it drops at iteration lr_step + 1 (base_model.py:155-165)."""
    trace = _lr_trace(_train_opt(lr_steps=[3, 5], lr_gamma=0.1), 8)
    for it, lrs in enumerate(trace, 1):
        k = sum(m <= it - 1 for m in (3, 5))
        assert lrs == pytest.approx([1e-4 * 0.1 ** k, 2e-4 * 0.1 ** k], rel=1e-12), (it, lrs)
    assert trace[2][0] == pytest.approx(1e-4) and trace[3][0] == pytest.approx(1e-5)


def test_warmup_is_linear_then_holds_the_last_warmup_lr():
    """Below warmup_iter the lr is initial x it / warmup_iter; from there the scheduler steps from the lr it finds
    (the reference's handling), so the lr holds initial x (warmup_iter - 1) / warmup_iter until a milestone."""
    trace = _lr_trace(_train_opt(lr_steps=[6], lr_gamma=0.5, warmup_iter=4), 8)
    for it in (1, 2, 3):
        assert trace[it - 1] == pytest.approx([1e-4 * it / 4, 2e-4 * it / 4], rel=1e-12)
    for it in (4, 5, 6):
        assert trace[it - 1] == pytest.approx([1e-4 * 3 / 4, 2e-4 * 3 / 4], rel=1e-12)
    for it in (7, 8):
        assert trace[it - 1] == pytest.approx([1e-4 * 3 / 8, 2e-4 * 3 / 8], rel=1e-12)


def test_other_lr_schemes_raise():
    from mmsr.models.ref_restoration_model import build_scheduler
    opt = torch.optim.Adam([torch.nn.Parameter(torch.zeros(1))], lr=1e-4)
    with pytest.raises(NotImplementedError, match='CosineAnnealingRestartLR'):
        build_scheduler(opt, _train_opt(lr_scheme='CosineAnnealingRestartLR'))


def _pil_down(img_bgr01, size):
    from PIL import Image
    rgb = (img_bgr01 * 255).astype(np.uint8)[..., ::-1]
    pil = Image.fromarray(np.ascontiguousarray(rgb)).resize((size, size), Image.BICUBIC)
    return np.asarray(pil)[..., ::-1].astype(np.float32) / 255.0


def _dihedral(img):
    """The 8 results of the flips / transpose the augmentation can apply, HWC."""
    out = []
    for h in (False, True):
        for v in (False, True):
            for t in (False, True):
                x = img[:, ::-1] if h else img
                x = x[::-1] if v else x
                out.append(x.transpose(1, 0, 2) if t else x)
    return out


def _bgr(t):
    return t.numpy().transpose(1, 2, 0)[..., ::-1]


def test_synthetic_train_sample_shapes_and_lq_is_pil_bicubic_of_the_crop():
    from mmsr.data import create_dataset
    ds = create_dataset({'name': 's', 'type': 'SyntheticRefDataset', 'phase': 'train', 'scale': 4, 'num': 3,
                         'gt_size': 96, 'in_size': 112, 'ref_size': 100, 'use_flip': True, 'use_rot': True})
    random.seed(3)
    s = ds[1]
    assert set(s) == {'img_in', 'img_in_lq', 'img_in_up', 'img_ref', 'img_ref_lq', 'img_ref_up'}
    shapes = {k: tuple(v.shape) for k, v in s.items()}
    assert shapes == {'img_in': (3, 96, 96), 'img_in_lq': (3, 24, 24), 'img_in_up': (3, 96, 96),
                      'img_ref': (3, 96, 96), 'img_ref_lq': (3, 24, 24), 'img_ref_up': (3, 96, 96)}
    assert all(v.dtype == torch.float32 for v in s.values())
    gt = _bgr(s['img_in'])
    assert np.array_equal(_bgr(s['img_in_lq']), _pil_down(gt, 24))
    assert np.array_equal(_bgr(s['img_ref_lq']), _pil_down(_bgr(s['img_ref']), 24))


def test_train_crop_is_a_window_of_the_input_under_one_of_the_eight_augmentations():
    from mmsr.data.ref_cufed_dataset import make_train_sample
    rng = np.random.default_rng(0)
    img = rng.random((40, 44, 3)).astype(np.float32)
    ref = rng.random((30, 30, 3)).astype(np.float32)
    for seed in range(6):
        random.seed(seed)
        gt = _bgr(make_train_sample(img, ref, 32, 4, True, True)['img_in'])
        hits = [(y, x) for y in range(40 - 32 + 1) for x in range(44 - 32 + 1)
                if any(np.array_equal(gt, d) for d in _dihedral(img[y:y + 32, x:x + 32]))]
        assert len(hits) == 1, (seed, hits)


def test_flips_and_rotation_act_alike_on_input_and_ref():
    """Input and Ref made from the same picture (the Ref at gt_size already, so its PIL resize is the identity and
    only its uint8 quantisation remains): every augmented pair stays pixel-aligned, and all 8 augmentations occur."""
    from mmsr.data.ref_cufed_dataset import make_train_sample
    rng = np.random.default_rng(1)
    pic = ((rng.integers(0, 256, (32, 32, 3)) + 0.5) / 255).astype(np.float32)
    seen = set()
    for seed in range(64):
        random.seed(seed)
        s = make_train_sample(pic, pic, 32, 4, True, True)
        gt, ref = _bgr(s['img_in']), _bgr(s['img_ref'])
        assert np.array_equal(np.round(ref * 255), np.floor(gt * 255)), seed
        assert torch.equal(s['img_in_lq'], s['img_ref_lq']) and torch.equal(s['img_in_up'], s['img_ref_up'])
        seen.add(next(i for i, d in enumerate(_dihedral(pic)) if np.array_equal(gt, d)))
    assert seen == set(range(8))
    random.seed(0)
    plain = make_train_sample(pic, pic, 32, 4, False, False)
    assert np.array_equal(_bgr(plain['img_in']), pic)


def test_dist_iter_sampler_shards_are_disjoint_and_cover_the_enlarged_set():
    from mmsr.data.data_sampler import DistIterSampler

    class _Len:
        def __len__(self):
            return 10

    for world, ratio in ((1, 1), (4, 3), (3, 7)):
        shards = [list(DistIterSampler(_Len(), world, r, ratio)) for r in range(world)]
        total = -(-10 * ratio // world) * world
        assert all(len(s) == total // world for s in shards)
        got = collections.Counter(i for s in shards for i in s)
        want = collections.Counter(v % 10 for v in range(total))
        assert got == want, (world, ratio)
        # the shards are slices of ONE permutation of the enlarged set: dealt back together they give it
        g = torch.Generator()
        g.manual_seed(0)
        perm = torch.randperm(total, generator=g).tolist()
        dealt = [None] * total
        for r, s in enumerate(shards):
            dealt[r::world] = s
        assert dealt == [v % 10 for v in perm]
    a = DistIterSampler(_Len(), 2, 1, 5)
    first = list(a)
    a.set_epoch(1)
    assert list(a) != first
    a.set_epoch(0)
    assert list(a) == first


def test_train_loader_batches_per_gpu_and_repeats_with_the_seed():
    from mmsr.data import create_dataloader, create_dataset
    dopt = {'name': 's', 'type': 'SyntheticRefDataset', 'phase': 'train', 'scale': 4, 'num': 5, 'gt_size': 32,
            'in_size': 40, 'ref_size': 36, 'use_flip': True, 'use_rot': True, 'batch_size': 2, 'n_workers': 2,
            'dataset_enlarge_ratio': 3}
    ds = create_dataset(dopt)

    def first_batches(seed):
        loader = create_dataloader(ds, dopt, seed=seed)
        loader.sampler.set_epoch(0)
        assert len(loader) == 15 // 2          # drop_last
        it = iter(loader)
        out = [next(it) for _ in range(3)]
        del it
        return out

    a, b, c = first_batches(10), first_batches(10), first_batches(11)
    assert tuple(a[0]['img_in'].shape) == (2, 3, 32, 32) and tuple(a[0]['img_in_lq'].shape) == (2, 3, 8, 8)
    assert all(torch.equal(x[k], y[k]) for x, y in zip(a, b) for k in x)
    assert not all(torch.equal(x['img_in'], y['img_in']) for x, y in zip(a, c))


@pytest.mark.parametrize('option', ['train.perceptual_opt', 'train.style_opt', 'train.texture_opt', 'train.gan_type',
                                    'network_d', 'path.pretrain_model_d'])
def test_out_of_scope_options_raise_naming_the_option(option):
    from mmsr.models.ref_restoration_model import RefRestorationModel
    from mmsr.utils.options import parse
    opt = parse(FIXTURE, is_train=True)
    section, _, key = option.rpartition('.')
    holder = opt[section] if section else opt
    holder[key] = {'type': 'x'} if key in ('perceptual_opt', 'style_opt', 'texture_opt', 'network_d') else 'x'
    with pytest.raises(NotImplementedError, match=option.replace('.', r'\.')):
        RefRestorationModel(opt)


def test_pixel_loss_weight_and_reduction():
    from mmsr.models.ref_restoration_model import PixelLoss
    a, b = torch.randn(2, 3, 4, 4, dtype=torch.float64), torch.randn(2, 3, 4, 4, dtype=torch.float64)
    assert float(PixelLoss('L1Loss', 2.0)(a, b)) == pytest.approx(2 * float((a - b).abs().mean()), rel=1e-12)
    assert float(PixelLoss('MSELoss', 1.0, 'sum')(a, b)) == pytest.approx(float(((a - b) ** 2).sum()), rel=1e-12)
    with pytest.raises(NotImplementedError, match='CharbonnierLoss'):
        PixelLoss('CharbonnierLoss')
