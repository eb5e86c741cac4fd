"""Training CLI with the reference's interface (mmsr/train.py), for the pixel-loss stage of the restoration
network (options/train/stage3_restoration_mse.yml):

    python mmsr/train.py -opt options/train/stage3_restoration_mse.yml [--launcher none|pytorch]

`--launcher pytorch` runs one process per GPU under torchrun (NCCL, DistributedDataParallel around net_g); each
rank loads its `rank::world` share of every batch.  `path.resume_state` continues from a training state: net_g
from models/net_g_<iter>.pth, optimizer and scheduler from the state."""
import argparse
import logging
import math
import os
import os.path as osp
import random
import sys
import time

sys.path.insert(0, osp.dirname(osp.dirname(osp.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mmsr.data import create_dataloader, create_dataset  # noqa: E402
from mmsr.models import create_model  # noqa: E402
from mmsr.utils.options import dict2str, dict_to_nonedict, parse  # noqa: E402


def set_random_seed(seed):
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)


def make_exp_dirs(opt):
    """util.py:47-72: an existing experiment directory is renamed aside, then every path directory is made."""
    root = opt['path']['experiments_root']
    if osp.exists(root):
        new = root + '_archived_' + time.strftime('%Y%m%d_%H%M%S')
        print(f'Path already exists. Rename it to {new}', flush=True)
        os.rename(root, new)
    for key, path in opt['path'].items():
        if key in ('experiments_root', 'models', 'training_state', 'log', 'visualization'):
            os.makedirs(path, exist_ok=True)


def check_resume(opt, resume_iter):
    """util.py:20-44: a resumed run takes net_g from the checkpoint saved with the training state."""
    if opt['path'].get('pretrain_model_g'):
        logging.getLogger('base').warning('pretrain_model_g will be ignored during resuming.')
    opt['path']['pretrain_model_g'] = osp.join(opt['path']['models'], f'net_g_{resume_iter}.pth')


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('-opt', type=str, required=True, help='Path to option YAML file.')
    parser.add_argument('--launcher', choices=['none', 'pytorch'], default='none', help='job launcher')
    parser.add_argument('--local_rank', type=int, default=0)
    args = parser.parse_args(argv)
    opt = parse(args.opt, is_train=True)

    if args.launcher == 'none':
        opt['dist'] = False
        rank = 0
        print('Disabled distributed training.', flush=True)
        if torch.cuda.is_available():
            ids = opt.get('gpu_ids') or [0]
            torch.cuda.set_device(int(ids[0]) % torch.cuda.device_count())
    else:
        opt['dist'] = True
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', args.local_rank)))
        torch.distributed.init_process_group(backend='nccl')
        rank = torch.distributed.get_rank()

    resume_state = None
    if opt['path'].get('resume_state'):
        resume_state = torch.load(opt['path']['resume_state'], map_location='cpu', weights_only=False)
        check_resume(opt, resume_state['iter'])
    if rank == 0 and resume_state is None:
        make_exp_dirs(opt)
    if opt['dist']:
        torch.distributed.barrier()

    logger = logging.getLogger('base')
    if not logger.handlers:
        logger.setLevel(logging.INFO)
        if rank == 0:
            logger.addHandler(logging.StreamHandler())
            logger.addHandler(logging.FileHandler(osp.join(
                opt['path']['log'], f"train_{opt['name']}_{time.strftime('%Y%m%d_%H%M%S')}.log")))
    logger.info(dict2str(opt))
    opt = dict_to_nonedict(opt)

    seed = opt['train']['manual_seed']
    if seed is None:
        seed = random.randint(1, 10000)
    logger.info(f'Random seed: {seed}')
    set_random_seed(seed)

    train_loader = val_loader = None
    for phase, dataset_opt in opt['datasets'].items():
        if phase == 'train':
            train_set = create_dataset(dataset_opt)
            train_loader = create_dataloader(train_set, dataset_opt, seed=seed)
            iters_per_epoch = len(train_loader)
            if iters_per_epoch == 0:
                raise ValueError('the train set is smaller than one batch per GPU')
            total_iters = int(opt['train']['niter'])
            total_epochs = int(math.ceil(total_iters / iters_per_epoch))
            logger.info(f'Number of train images: {len(train_set)}, iters per epoch: {iters_per_epoch}')
            logger.info(f'Total epochs needed: {total_epochs} for iters {total_iters}')
        elif phase == 'val':
            val_set = create_dataset(dataset_opt)
            val_loader = create_dataloader(val_set, dataset_opt, dist=opt['dist'])
            logger.info(f"Number of val images in {dataset_opt['name']}: {len(val_set)}")
        else:
            raise NotImplementedError(f'Phase {phase} is not recognized.')
    if train_loader is None:
        raise ValueError('datasets.train is missing')

    model = create_model(opt)
    if resume_state:
        logger.info(f"Resuming training from epoch: {resume_state['epoch']}, iter: {resume_state['iter']}.")
        start_epoch, current_iter = resume_state['epoch'], resume_state['iter']
        model.resume_training(resume_state)
    else:
        start_epoch, current_iter = 0, 0

    val_freq = int(opt['val']['val_freq']) if opt['val'] and opt['val']['val_freq'] else 0
    print_freq = int(opt['logger']['print_freq'] or 1)
    save_freq = int(opt['logger']['save_checkpoint_freq'] or 0)
    logger.info(f'Start training from epoch: {start_epoch}, iter: {current_iter}')
    epoch = start_epoch
    t_start = time.time()
    for epoch in range(start_epoch, total_epochs + 1):
        if current_iter >= total_iters:
            break
        train_loader.sampler.set_epoch(epoch)
        t_data = time.time()
        for train_data in train_loader:
            data_time = time.time() - t_data
            current_iter += 1
            if current_iter > total_iters:
                break
            model.update_learning_rate(current_iter, warmup_iter=opt['train']['warmup_iter'] or -1)
            model.feed_data(train_data)
            model.optimize_parameters(current_iter)
            iter_time = time.time() - t_data
            if current_iter % print_freq == 0:
                log = model.get_current_log()
                eta = (time.time() - t_start) / max(1, current_iter - (resume_state or {}).get('iter', 0)) * \
                    (total_iters - current_iter)
                msg = (f"[{opt['name'][:5]}..][epoch:{epoch:3d}, iter:{current_iter:8,d}, lr:(" +
                       ''.join(f'{v:.3e},' for v in model.get_current_learning_rate()) +
                       f')] [eta: {int(eta)}s, time: {iter_time:.3f}, data_time: {data_time:.3f}] ' +
                       ' '.join(f'{k}: {v:.4e}' for k, v in log.items()))
                logger.info(msg)
            if val_loader is not None and val_freq and current_iter % val_freq == 0:
                model.validation(val_loader, current_iter, None, bool(opt['val']['save_img']))
            if save_freq and current_iter % save_freq == 0:
                logger.info('Saving models and training states.')
                model.save(epoch, current_iter)
            t_data = time.time()

    logger.info('End of training.')
    logger.info('Saving the latest model.')
    model.save(epoch=-1, current_iter=-1)
    if opt['dist']:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == '__main__':
    main()
