"""`RefRestorationModel` (reference: mmsr/models/ref_restoration_model.py, base_model.py, sr_model.py):
owns net_extractor / net_map / net_g, loads the reference's checkpoints strictly, `feed_data` / `test` /
`get_current_visuals` / `validation`, and with `is_train` the pixel-loss training of net_g (stage 3,
options/train/stage3_restoration_mse.yml): Adam over the reference's four parameter groups, MultiStepLR with
linear warm-up, L1 / MSE pixel loss, checkpoints and training states in the reference's layout.

Execution differences from the reference (SURVEY.md §8f N1): one process per GPU instead of
nn.DataParallel (DistributedDataParallel around net_g when training with `dist`); no per-image
`torch.cuda.empty_cache()`; validation can be rank-sharded with `torch.distributed` (the reference's dist
validation is broken, sr_model.py:160-162) and metrics are all-gathered at the end.  In training the frozen
extractor and net_map run under no_grad, and the reference's stage-3 model builds its schedulers before its
generator optimizer exists (ref_restoration_model.py:44-87 after sr_model.py:38-39), so there `lr_steps`
never take effect; here they do.  GAN / perceptual / style / texture options raise NotImplementedError."""
import logging
import os
import os.path as osp
from collections import OrderedDict

import torch
import torch.nn.functional as F

from c2m_b200.dist import gather_rows
from mmsr.models import networks
from mmsr.utils import metrics, metrics_torch
from mmsr.utils.util import tensor2img

logger = logging.getLogger('base')


# options of losses and networks this build does not train (the GAN stage, perceptual / style / texture losses)
_OUT_OF_SCOPE = (('train', 'perceptual_opt'), ('train', 'style_opt'), ('train', 'texture_opt'), ('train', 'gan_type'),
                 (None, 'network_d'), ('path', 'pretrain_model_d'))


def check_train_scope(opt):
    """Raise NotImplementedError naming the first option that needs a loss or network outside pixel-loss training."""
    for section, key in _OUT_OF_SCOPE:
        holder = opt if section is None else (opt.get(section) or {})
        if holder.get(key):
            name = key if section is None else f'{section}.{key}'
            raise NotImplementedError(f'option {name} needs a loss or network outside pixel-loss training of net_g '
                                      '(the GAN stage and the perceptual, style and texture losses are not built)')


def param_groups(net_g):
    """The reference's split of net_g's trainable parameters (ref_restoration_model.py:54-68): names containing
    'offset' and 'small' -> relu3_offset, 'offset' and 'medium' -> relu2_offset, other 'offset' names -> offset,
    the rest -> g.  Returns OrderedDict group -> [(name, parameter)] in the reference's optimizer order."""
    groups = OrderedDict((k, []) for k in ('g', 'offset', 'relu3_offset', 'relu2_offset'))
    for name, v in net_g.named_parameters():
        if not v.requires_grad:
            continue
        if 'offset' in name:
            groups['relu3_offset' if 'small' in name else 'relu2_offset' if 'medium' in name else 'offset'].append((name, v))
        else:
            groups['g'].append((name, v))
    return groups


def build_optimizer(net_g, train_opt):
    """Adam over param_groups with lr_g / lr_offset / lr_relu3_offset / lr_relu2_offset, weight_decay_g, beta_g
    (ref_restoration_model.py:70-85)."""
    g = param_groups(net_g)
    lrs = {'offset': train_opt['lr_offset'], 'relu3_offset': train_opt['lr_relu3_offset'],
           'relu2_offset': train_opt['lr_relu2_offset']}
    return torch.optim.Adam([{'params': [p for _, p in ps], **({'lr': float(lrs[k])} if k in lrs else {})}
                             for k, ps in g.items()],
                            lr=float(train_opt['lr_g']), weight_decay=float(train_opt.get('weight_decay_g') or 0),
                            betas=tuple(float(b) for b in train_opt.get('beta_g') or (0.9, 0.999)))


def build_scheduler(optimizer, train_opt):
    """`lr_scheme: MultiStepLR` (base_model.py:77-86: MultiStepRestartLR without restarts, which is torch's
    MultiStepLR): every group's lr times lr_gamma at each of lr_steps."""
    scheme = train_opt.get('lr_scheme') or 'MultiStepLR'
    if scheme != 'MultiStepLR':
        raise NotImplementedError(f'lr_scheme {scheme} is not implemented (MultiStepLR is)')
    return torch.optim.lr_scheduler.MultiStepLR(optimizer, list(train_opt.get('lr_steps') or []),
                                                gamma=float(train_opt.get('lr_gamma') or 0.1))


def update_learning_rate(optimizers, schedulers, current_iter, warmup_iter=-1):
    """base_model.py:155-177: step the schedulers from the second iteration on; below warmup_iter every group's lr
    is its initial lr x current_iter / warmup_iter.  As there, the scheduler steps from the lr it finds, so after a
    warm-up the lr stays at the last warm-up value (initial x (warmup_iter - 1) / warmup_iter) until a step."""
    if current_iter > 1:
        for s in schedulers:
            s.step()
    if warmup_iter is not None and current_iter < warmup_iter:
        for o in optimizers:
            for g in o.param_groups:
                g['lr'] = g['initial_lr'] / warmup_iter * current_iter


class PixelLoss(torch.nn.Module):
    """`pixel_criterion` L1Loss / MSELoss of losses.py:30-83 without element weights: loss_weight x the
    elementwise loss reduced by 'mean' or 'sum'."""

    def __init__(self, criterion, loss_weight=1.0, reduction='mean'):
        super().__init__()
        fns = {'L1Loss': F.l1_loss, 'MSELoss': F.mse_loss}
        if criterion not in fns:
            raise NotImplementedError(f'pixel_criterion {criterion} is not implemented (L1Loss, MSELoss are)')
        if reduction not in ('mean', 'sum'):
            raise ValueError(f"reduction must be 'mean' or 'sum', got {reduction!r}")
        self.fn, self.loss_weight, self.reduction = fns[criterion], float(loss_weight), reduction

    def forward(self, pred, target):
        return self.loss_weight * self.fn(pred, target, reduction=self.reduction)


def _bare(net):
    return net.module if isinstance(net, torch.nn.parallel.DistributedDataParallel) else net


class RefRestorationModel:

    def __init__(self, opt):
        self.opt = opt
        self.is_train = bool(opt.get('is_train'))
        if self.is_train:
            check_train_scope(opt)
        if not torch.cuda.is_available():
            raise RuntimeError('RefRestorationModel needs a CUDA device: the H100 hot path has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device())
        path = opt.get('path') or {}
        # parity is stated against the reference's fp32 arithmetic: any convolution that falls back to cuDNN
        # (maps below the tensor-core kernel's tile size, C2M_FAST_CONV=0) must not run in TF32 (torch's default)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        # net_map's VGG19 is never loaded from a checkpoint in the reference: it is built with ImageNet weights
        # (vgg_arch.py:103-104).  Optional `path.pretrain_model_vgg` names a local torchvision checkpoint.
        if path.get('pretrain_model_vgg') and opt.get('network_map') is not None:
            opt['network_map'].setdefault('vgg_pretrained_path', path['pretrain_model_vgg'])
        self.net_g = networks.define_net_g(opt).to(self.device).eval()
        self.net_map = networks.define_net_map(opt).to(self.device).eval()
        self.net_extractor = networks.define_net_extractor(opt).to(self.device).eval()
        strict = path.get('strict_load', True)
        for key in ('pretrain_model_feature_extractor', 'pretrain_model_g'):
            if not path.get(key):
                logger.warning(f'path.{key} is not set: the network keeps its random initial weights.')
        if path.get('pretrain_model_feature_extractor'):
            self.load_network(self.net_extractor, path['pretrain_model_feature_extractor'], strict)
        if path.get('pretrain_model_g'):
            self.load_network(self.net_g, path['pretrain_model_g'], strict)
        if self.is_train:
            self.init_training_settings()

    # -- training (ref_restoration_model.py:44-110, 186-269, base_model.py:136-307)
    def init_training_settings(self):
        train_opt = self.opt['train']
        if self.opt.get('use_tb_logger'):
            logger.warning('use_tb_logger is set: TensorBoard logging is not built, the run logs to its text log only.')
        for net in (self.net_extractor, self.net_map):
            net.eval().requires_grad_(False)
        self.net_g.train()
        if self.opt.get('dist'):
            self.net_g = torch.nn.parallel.DistributedDataParallel(self.net_g, device_ids=[self.device.index])
        if not float(train_opt.get('pixel_weight') or 0) > 0:
            raise ValueError('pixel_weight must be > 0: the pixel loss is the only loss trained here')
        self.cri_pix = PixelLoss(train_opt.get('pixel_criterion') or 'L1Loss', train_opt['pixel_weight'],
                                 train_opt.get('reduction') or 'mean')
        self.net_g_pretrain_steps = int(train_opt.get('net_g_pretrain_steps') or 0)
        self.net_d_steps = int(train_opt.get('net_d_steps') or 1)
        self.net_d_init_steps = int(train_opt.get('net_d_init_steps') or 0)
        self.optimizer_g = build_optimizer(_bare(self.net_g), train_opt)
        self.optimizers = [self.optimizer_g]
        self.schedulers = [build_scheduler(self.optimizer_g, train_opt)]
        self.log_dict = OrderedDict()

    def optimize_parameters(self, step):
        """One step of net_g on the pixel loss (ref_restoration_model.py:192-269 without a discriminator): the
        frozen extractor and net_map run forward under no_grad.  As in the reference the loss is logged as l_pix
        up to net_g_pretrain_steps and as l_g_pix after, where net_d_steps / net_d_init_steps gate the update."""
        with torch.no_grad():
            self.features = self.net_extractor(self.match_img_in, self.img_ref)
            self.pre_offset, self.img_ref_feat = self.net_map(self.features, self.img_ref)
        pretrain = step <= self.net_g_pretrain_steps
        k = step - self.net_g_pretrain_steps
        if not pretrain and not (k % self.net_d_steps == 0 and k > self.net_d_init_steps):
            return
        self.output = self.net_g(self.img_in_lq, self.pre_offset, self.img_ref_feat)
        self.optimizer_g.zero_grad()
        l_pix = self.cri_pix(self.output, self.gt)
        l_pix.backward()
        self.optimizer_g.step()
        self.log_dict['l_pix' if pretrain else 'l_g_pix'] = l_pix.detach()     # read on the host only when logged

    def update_learning_rate(self, current_iter, warmup_iter=-1):
        update_learning_rate(self.optimizers, self.schedulers, current_iter, warmup_iter)

    def get_current_learning_rate(self):
        return [g['lr'] for g in self.optimizer_g.param_groups]

    def get_current_log(self):
        return OrderedDict((k, float(v)) for k, v in self.log_dict.items())

    def _rank0(self):
        return not (torch.distributed.is_available() and torch.distributed.is_initialized()) or \
            torch.distributed.get_rank() == 0

    def save(self, epoch, current_iter):
        """net_g_<iter>.pth (net_g_latest.pth for iter -1) and, for iter != -1, training_state/<iter>.state with the
        epoch, the iteration and the optimizer and scheduler states (base_model.py:185-290); rank 0 writes."""
        if not self._rank0():
            return
        self.save_network(self.net_g, 'net_g', 'latest' if current_iter == -1 else current_iter)
        if current_iter != -1:
            state = {'epoch': epoch, 'iter': current_iter, 'optimizers': [o.state_dict() for o in self.optimizers],
                     'schedulers': [s.state_dict() for s in self.schedulers]}
            torch.save(state, osp.join(self.opt['path']['training_state'], f'{current_iter}.state'))

    def resume_training(self, resume_state):
        """Load the optimizer and scheduler states of a training state (base_model.py:292-307); net_g's weights come
        from its checkpoint (`path.pretrain_model_g`)."""
        if len(resume_state['optimizers']) != len(self.optimizers) or \
                len(resume_state['schedulers']) != len(self.schedulers):
            raise ValueError('the training state holds a different number of optimizers or schedulers')
        for o, sd in zip(self.optimizers, resume_state['optimizers']):
            o.load_state_dict(sd)
        for s, sd in zip(self.schedulers, resume_state['schedulers']):
            s.load_state_dict(sd)

    # -- checkpoint I/O (base_model.py:245-265: strips DataParallel's `module.` prefix)
    def load_network(self, net, load_path, strict=True):
        net = _bare(net)
        logger.info(f'Loading {net.__class__.__name__} model from {load_path}.')
        sd = torch.load(load_path, map_location='cpu')
        sd = OrderedDict((k[7:] if k.startswith('module.') else k, v) for k, v in sd.items())
        net.load_state_dict(sd, strict=strict)

    def save_network(self, net, net_label, current_iter):
        save_path = osp.join(self.opt['path']['models'], f'{net_label}_{current_iter}.pth')
        torch.save(OrderedDict((k, v.cpu()) for k, v in _bare(net).state_dict().items()), save_path)

    # -- data / forward (ref_restoration_model.py:186-190, 271-287)
    def feed_data(self, data):
        nb = dict(non_blocking=True)
        self.img_in_lq = data['img_in_lq'].to(self.device, **nb)
        self.img_ref = data['img_ref'].to(self.device, **nb)
        if 'img_in' in data:
            self.gt = data['img_in'].to(self.device, **nb)
        self.match_img_in = data['img_in_up'].to(self.device, **nb)

    @torch.no_grad()
    def test(self):
        self.features = self.net_extractor(self.match_img_in, self.img_ref)
        self.pre_offset, self.img_ref_feat = self.net_map(self.features, self.img_ref)
        # the bare net_g: a forward through DistributedDataParallel would take part in its collectives, and the ranks
        # of a sharded validation run different numbers of batches
        self.output = _bare(self.net_g)(self.img_in_lq, self.pre_offset, self.img_ref_feat)

    def get_current_visuals(self):
        out = OrderedDict(img_in_lq=self.img_in_lq.detach().cpu(), rlt=self.output.detach().cpu())
        if hasattr(self, 'gt'):
            out['gt'] = self.gt.detach().cpu()
        return out

    # -- validation (ref_restoration_model.py:295-370): rank-sharded, batched, host work off the GPU's critical path
    # packed-split activations are fp16 pairs: |x * 2^sa| must stay below 65504 (c2m_b200.ops.PSA)
    _NONFINITE = ('non-finite SR output for {}: an activation left the fp16 range of the packed-split layout '
                  '(ops.suggest_sa / PSA.sa) or the inputs were not finite')

    def _png_name(self, meta):
        return f"{meta['name']}_{self.opt['name']}" + (f"_{self.opt['suffix']}" if self.opt.get('suffix') else '') + '.png'

    def _save_image(self, sr, meta, save_dir):
        """PNG only (the metrics were computed on the GPU)."""
        import cv2
        sr_img = tensor2img(sr)
        if meta['padding']:
            oh, ow = meta['original_size']
            sr_img = sr_img[:oh, :ow]
        cv2.imwrite(osp.join(save_dir, self._png_name(meta)), sr_img)
        return None

    def _score_image(self, sr, gt, meta, crop, save_dir):
        """CPU post-processing of one image: tensor2img, un-pad, PNG, PSNR / PSNR_Y / SSIM_Y (reference :306-360)."""
        if not bool(torch.isfinite(sr).all()):
            raise RuntimeError(self._NONFINITE.format(meta['name']))
        sr_img, gt_img = tensor2img([sr, gt])
        if meta['padding']:
            oh, ow = meta['original_size']
            sr_img, gt_img = sr_img[:oh, :ow], gt_img[:oh, :ow]
        if save_dir is not None:
            import cv2
            cv2.imwrite(osp.join(save_dir, self._png_name(meta)), sr_img)
        psnr = metrics.psnr(sr_img, gt_img, crop_border=crop)
        sr_y = metrics.bgr2ycbcr(sr_img / 255., only_y=True)
        gt_y = metrics.bgr2ycbcr(gt_img / 255., only_y=True)
        psnr_y = metrics.psnr(sr_y * 255, gt_y * 255, crop_border=crop)
        ssim_y = metrics.ssim(sr_y * 255, gt_y * 255, crop_border=crop)
        logger.info(f"# img {meta['name']} # PSNR: {psnr:.4e} # PSNR_Y: {psnr_y:.4e} # SSIM_Y: {ssim_y:.4e}.")
        return (meta['index'], psnr, psnr_y, ssim_y)

    def validation(self, dataloader, current_iter, tb_logger=None, save_img=False, post_workers=None,
                   metrics_device=None):
        """The loader hands this rank only ITS pairs (ShardedEvalSampler), batched by shape; per batch the GPU runs
        one forward.  `metrics_device` (`opt['metrics_device']`, default 'cuda'): 'cuda' scores the batch where it is
        (`utils/metrics_torch.py`: same definitions and dtypes as the host metrics, equal to ~1e-14) and nothing
        returns to the host but four numbers per image; 'cpu' is the reference's own arithmetic (`utils/metrics.py`,
        cv2) on a thread pool fed through a pinned ring with an async D2H copy.  PNGs (`save_img`) always go through
        the pinned ring + thread pool.  The ranks' metric rows are all-gathered at the end."""
        import time
        from concurrent.futures import ThreadPoolExecutor
        dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
        rank = torch.distributed.get_rank() if dist_on else 0
        crop = self.opt.get('crop_border')
        if crop is None:
            crop = self.opt.get('scale', 4)
        metrics_device = metrics_device or self.opt.get('metrics_device') or 'cuda'
        if metrics_device not in ('cuda', 'cpu'):
            raise ValueError(f"metrics_device must be 'cuda' or 'cpu', got {metrics_device!r}")
        on_gpu = metrics_device == 'cuda'
        dataset_name = dataloader.dataset.opt['name']
        save_dir = None
        if save_img:
            save_dir = osp.join(self.opt['path']['visualization'], dataset_name)
            os.makedirs(save_dir, exist_ok=True)
        host_post = save_img or not on_gpu
        batches = getattr(getattr(dataloader, 'batch_sampler', None), 'batches', None)
        pool = ThreadPoolExecutor(max_workers=int(post_workers or self.opt.get('post_workers') or 4))
        # the post-processing threads are the parallelism: torch / OpenCV intra-op pools on top of them oversubscribe
        # the host (measured: a 1.2 M-element clamp took 57 ms instead of 1 ms)
        prev_threads = torch.get_num_threads()
        torch.set_num_threads(1)
        try:
            import cv2
            cv2.setNumThreads(1)
        except Exception:
            pass
        ring, futures = [], []          # ring of (pinned buffer, in-flight futures using it)
        gpu_rows, metas, spans = [], [], []
        depth = 3
        t_load = t_gpu = 0.0
        n_img = 0
        t0 = time.perf_counter()
        it = iter(dataloader)
        bi = 0
        while True:
            tl = time.perf_counter()
            try:
                val_data = next(it)
            except StopIteration:
                break
            t_load += time.perf_counter() - tl
            tg = time.perf_counter()
            ev0 = torch.cuda.Event(enable_timing=True)
            ev0.record()
            # host metrics: the ground truth stays on the host (the reference ships it to the GPU and back)
            self.feed_data({k: v for k, v in val_data.items() if torch.is_tensor(v) and (on_gpu or k != 'img_in')})
            stage = val_data.get('_slot')
            if stage is not None:       # PairBatcher staging buffers: reusable once these H2D copies are done
                stage['event'] = torch.cuda.Event()
                stage['event'].record()
            self.test()
            out = self.output
            n = out.shape[0]
            idxs = batches[bi] if batches is not None else list(range(n_img, n_img + n))
            pad = val_data.get('padding')
            osz = val_data.get('original_size')
            bmeta = [{'index': int(idxs[k]), 'name': osp.splitext(osp.basename(val_data['lq_path'][k]))[0],
                      'padding': bool(pad[k]) if pad is not None else False,
                      'original_size': tuple(int(v) for v in osz[k][:2]) if osz is not None else None}
                     for k in range(n)]
            if on_gpu:
                for k, meta in enumerate(bmeta):
                    gpu_rows.append(metrics_torch.score_image(
                        out[k], self.gt[k], crop, meta['original_size'] if meta['padding'] else None))
                metas += bmeta
            if host_post:
                # pinned slot: reuse the oldest buffer of this shape once its consumers are done
                slot = None
                if len(ring) >= depth:
                    buf, futs = ring.pop(0)
                    for f in futs:
                        f.result()
                    if buf.shape == out.shape:
                        slot = buf
                if slot is None:
                    slot = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
                slot.copy_(out, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                gts = None if on_gpu else val_data['img_in']
                if gts is not None and stage is not None:
                    gts = gts.clone()       # the staging slot is recycled after its H2D copies; the pool reads GT later
                futs = []
                for k, meta in enumerate(bmeta):
                    def job(k=k, meta=meta, ev=ev, slot=slot, gts=gts):
                        ev.synchronize()
                        if gts is None:
                            return self._save_image(slot[k], meta, save_dir)
                        return self._score_image(slot[k], gts[k], meta, crop, save_dir)
                    futs.append(pool.submit(job))
                ring.append((slot, futs))
                futures += futs
            ev1 = torch.cuda.Event(enable_timing=True)
            ev1.record()
            spans.append((ev0, ev1))
            t_gpu += time.perf_counter() - tg
            n_img += n
            bi += 1
        rows = [f.result() for f in futures]
        pool.shutdown()
        torch.set_num_threads(prev_threads)
        if on_gpu:
            t = torch.stack(gpu_rows) if gpu_rows else torch.zeros(0, 4, dtype=torch.float64, device=self.device)
            host = t.cpu()              # the one synchronising read of the validation
            for meta, (p, py, sy, fin) in zip(metas, host.tolist()):
                if not fin:
                    raise RuntimeError(self._NONFINITE.format(meta['name']))
                logger.info(f"# img {meta['name']} # PSNR: {p:.4e} # PSNR_Y: {py:.4e} # SSIM_Y: {sy:.4e}.")
            t = torch.cat([torch.tensor([m['index'] for m in metas], dtype=torch.float64,
                                        device=self.device)[:, None], t[:, :3]], 1)
        else:
            t = torch.tensor(rows, dtype=torch.float64, device=self.device).reshape(-1, 4)
        torch.cuda.synchronize(self.device)
        wall = time.perf_counter() - t0
        gpu_busy = sum(a.elapsed_time(b) for a, b in spans) * 1e-3      # H2D + forward (+ metrics) per batch, on the device
        t = gather_rows(t)
        avg = t[:, 1:].mean(0).tolist() if t.numel() else [float('nan')] * 3
        if rank == 0:
            logger.info(f'# Validation {dataset_name} # PSNR: {avg[0]:.4e} # PSNR_Y: {avg[1]:.4e} # SSIM_Y: {avg[2]:.4e}.')
            if tb_logger:
                for k, v in zip(('psnr', 'psnr_y', 'ssim_y'), avg):
                    tb_logger.add_scalar(k, v, current_iter)
        self.last_validation = {'psnr': avg[0], 'psnr_y': avg[1], 'ssim_y': avg[2], 'n': int(t.shape[0]),
                                'rank_images': n_img, 'rank_wall_s': wall, 'rank_loader_wait_s': t_load,
                                'rank_submit_s': t_gpu, 'rank_gpu_busy_s': gpu_busy, 'metrics_device': metrics_device}
        return self.last_validation
