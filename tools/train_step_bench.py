"""Stage-3 training iterations per second of `RefRestorationModel` on one GPU (batch 9, GT 160: LR 40x40, Ref
160x160, synthetic data, the restoration network trained with the L1 pixel loss, extractor and net_map frozen).

Legs, alternated round by round in one process:
  library      every convolution on the tensor-core 3x3 kernel (forward, dX, dW), every DCN on the tensor-core DCN
  cudnn_ext    the same step with C2M_FAST_CONV=0 C2M_DCN_TC=0: cuDNN fp32 with TF32 off and `_ext`'s CUDA-core DCN
each with the batches already on the GPU (loader excluded: a ring of pre-made batches) and, for the library leg, from
the train loader (`n_workers` decoding workers, loader included).  A step is timed from its first enqueue to a device
synchronise.  Prints the card name and power limit and one JSON line; `--out` also writes it to a file.

    python tools/train_step_bench.py [--steps 20] [--warmup 3] [--rounds 3] [--workers 6] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'c2-matching_b200'), os.path.join(ROOT, 'tests', 'golden')):
    if p not in sys.path:
        sys.path.insert(0, p)
os.environ.setdefault('C2M_VGG_PRETRAINED', '0')

import torch  # noqa: E402

BATCH, GT = 9, 160


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the number is still a number without it, but say so
        q = f'nvidia-smi unavailable ({e})'
    return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q}


def model_opt(tmp):
    return {'name': 'train_step_bench', 'suffix': None, 'scale': 4, 'crop_border': None, 'dist': False,
            'is_train': True,
            'network_g': {'type': 'RestorationNet', 'ngf': 64, 'n_blocks': 16, 'groups': 8},
            'network_map': {'type': 'CorrespondenceGenerationArch', 'patch_size': 3, 'stride': 1,
                            'vgg_layer_list': ['relu1_1', 'relu2_1', 'relu3_1'], 'vgg_type': 'vgg19',
                            'vgg_pretrained': False},
            'network_extractor': {'type': 'ContrasExtractorSep'},
            'train': {'lr_g': 1e-4, 'lr_offset': 1e-4, 'lr_relu2_offset': 1e-5, 'lr_relu3_offset': 1e-6,
                      'weight_decay_g': 0, 'beta_g': [0.9, 0.999], 'lr_scheme': 'MultiStepLR', 'niter': 255000,
                      'warmup_iter': -1, 'lr_steps': [72545, 211040], 'lr_gamma': 0.1, 'pixel_criterion': 'L1Loss',
                      'pixel_weight': 1.0, 'manual_seed': 10},
            'path': {'models': tmp, 'training_state': tmp, 'visualization': tmp, 'strict_load': True}}


def dataset_opt(workers):
    # CUFED's training pairs: 160x160 inputs, Refs of varying size resized to 160x160
    return {'name': 'synth_train', 'type': 'SyntheticRefDataset', 'phase': 'train', 'scale': 4, 'num': 1024,
            'gt_size': GT, 'in_size': GT, 'ref_size': 180, 'use_flip': True, 'use_rot': True,
            'batch_size': BATCH, 'n_workers': workers, 'dataset_enlarge_ratio': 1000}


def set_leg(leg):
    lib = leg == 'library'
    os.environ['C2M_FAST_CONV'] = '1' if lib else '0'
    os.environ['C2M_DCN_TC'] = '1' if lib else '0'


def timed(model, batches, steps, it0):
    """seconds for `steps` iterations fed from the iterator `batches`, ending in a device synchronise."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(steps):
        model.update_learning_rate(it0 + k)
        model.feed_data(next(batches))
        model.optimize_parameters(it0 + k)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--workers', type=int, default=6)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_step_bench needs a CUDA device')
    import itertools

    import __graft_entry__ as g
    g.build()
    import bench
    from mmsr.data import create_dataloader, create_dataset
    from mmsr.models.ref_restoration_model import RefRestorationModel
    tmp = tempfile.mkdtemp(prefix='train_step_bench_')
    model = RefRestorationModel(model_opt(tmp))
    for net, sd in zip((model.net_extractor, model.net_map, model.net_g), bench.seeded_weights()):
        net.load_state_dict(sd, strict=True)
    dset = create_dataset(dataset_opt(a.workers))
    loader = create_dataloader(dset, dataset_opt(a.workers), seed=10)
    loader.sampler.set_epoch(0)
    ring = []
    for b in itertools.islice(iter(loader), 4):
        ring.append({k: v.to('cuda', non_blocking=True) for k, v in b.items()})
    ring_it = itertools.cycle(ring)
    loader_it = iter(loader)
    res = {'library': [], 'cudnn_ext': [], 'library_with_loader': []}
    it = 1
    for leg in ('library', 'cudnn_ext'):
        set_leg(leg)
        timed(model, ring_it, a.warmup, it)
        it += a.warmup
    set_leg('library')
    timed(model, loader_it, a.warmup, it)
    it += a.warmup
    for _ in range(a.rounds):
        for leg in ('library', 'cudnn_ext'):
            set_leg(leg)
            res[leg].append(a.steps / timed(model, ring_it, a.steps, it))
            it += a.steps
        set_leg('library')
        res['library_with_loader'].append(a.steps / timed(model, loader_it, a.steps, it))
        it += a.steps
    loss = model.get_current_log()
    out = {'workload': f'stage-3 training step, batch {BATCH}, GT {GT} (LR {GT // 4}x{GT // 4}, Ref {GT}x{GT})',
           'unit': 'iterations/s', 'card': card(), 'steps': a.steps, 'rounds': a.rounds, 'workers': a.workers,
           'last_loss': loss, 'runs': res,
           'median': {k: sorted(v)[len(v) // 2] for k, v in res.items()}}
    out['speedup_vs_cudnn_ext'] = out['median']['library'] / out['median']['cudnn_ext']
    print(f"card: {out['card']}")
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
