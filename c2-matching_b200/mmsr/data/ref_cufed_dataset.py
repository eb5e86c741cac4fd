"""`RefCUFEDDataset` (reference: mmsr/data/ref_cufed_dataset.py:13-170) plus a file-free synthetic
stand-in with the same sample dict.

Test phase, per pair: mod-crop both images to the scale, zero-pad both (bottom/right) to a common size
(:99-114), PIL-bicubic x1/4 then x4 (:119-134), BGR->RGB CHW float tensors (:145-166).
Train phase, per pair: the input cropped to `gt_size` (CUFED's training inputs already are 160x160, so the
reference never crops), the Ref PIL-bicubic resized to `gt_size` (:85-93), the same random flips / rotation on
both (:95-96, transforms.py:89-145), then the test phase's PIL-bicubic x1/4 and x4."""
import os
import os.path as osp
import random

import numpy as np
import torch
import torch.utils.data as data


def _mod_crop(img, scale):
    h, w = img.shape[:2]
    return img[:h - h % scale, :w - w % scale].copy()


def _pad_to(img, h, w):
    out = np.zeros((h, w, img.shape[2]), img.dtype)
    out[:img.shape[0], :img.shape[1]] = img
    return out


def _pil_resize_bgr(img01, size_wh):
    """float BGR [0,1] -> uint8 RGB -> PIL bicubic -> (float BGR [0,1], PIL image)."""
    from PIL import Image
    rgb = (img01 * 255).astype(np.uint8)[..., ::-1]
    return Image.fromarray(np.ascontiguousarray(rgb)).resize(size_wh, Image.BICUBIC)


def _to_tensor_rgb(x):
    return torch.from_numpy(np.ascontiguousarray(x[..., ::-1].transpose(2, 0, 1))).float()


def _pil_to_bgr(pil):
    return np.asarray(pil)[..., ::-1].astype(np.float32) / 255.0


def _degraded(img_in, img_ref, scale):
    """PIL-bicubic x1/4 of both images and x4 of the results (reference :118-143), as RGB CHW tensors."""
    from PIL import Image
    gh, gw = img_in.shape[:2]
    lq = (gw // scale, gh // scale)
    in_lq = _pil_resize_bgr(img_in, lq)
    ref_lq = _pil_resize_bgr(img_ref, lq)
    in_up, ref_up = in_lq.resize((gw, gh), Image.BICUBIC), ref_lq.resize((gw, gh), Image.BICUBIC)
    return {'img_in_lq': _to_tensor_rgb(_pil_to_bgr(in_lq)), 'img_in_up': _to_tensor_rgb(_pil_to_bgr(in_up)),
            'img_ref_lq': _to_tensor_rgb(_pil_to_bgr(ref_lq)), 'img_ref_up': _to_tensor_rgb(_pil_to_bgr(ref_up))}


def make_sample(img_in, img_ref, scale, path=''):
    """img_in / img_ref: float32 BGR HWC in [0,1] -> the reference's test-phase sample dict."""
    img_in, img_ref = _mod_crop(img_in, scale), _mod_crop(img_ref, scale)
    img_in_gt = img_in.copy()
    (ih, iw), (rh, rw) = img_in.shape[:2], img_ref.shape[:2]
    padding = (ih, iw) != (rh, rw)
    if padding:
        th, tw = max(ih, rh), max(iw, rw)
        img_in, img_ref = _pad_to(img_in, th, tw), _pad_to(img_ref, th, tw)
    deg = _degraded(img_in, img_ref, scale)
    return {'img_in': _to_tensor_rgb(img_in_gt), 'img_in_lq': deg['img_in_lq'], 'img_in_up': deg['img_in_up'],
            'img_ref': _to_tensor_rgb(img_ref), 'img_ref_lq': deg['img_ref_lq'], 'img_ref_up': deg['img_ref_up'],
            'lq_path': path, 'padding': padding, 'original_size': (ih, iw)}


def augment(imgs, hflip=True, rotation=True):
    """The same random horizontal flip, vertical flip and transpose on every HWC image (transforms.py:89-145:
    three draws from `random`, in this order, whatever is enabled)."""
    hflip = hflip and random.random() < 0.5
    vflip = rotation and random.random() < 0.5
    rot90 = rotation and random.random() < 0.5
    out = []
    for img in imgs:
        if hflip:
            img = img[:, ::-1]
        if vflip:
            img = img[::-1]
        if rot90:
            img = img.transpose(1, 0, 2)
        out.append(np.ascontiguousarray(img))
    return out


def make_train_sample(img_in, img_ref, gt_size, scale, use_flip, use_rot, path=''):
    """img_in / img_ref: float32 BGR HWC in [0,1] -> the reference's train-phase sample dict: `img_in` a random
    gt_size crop of the input (drawn from `random` only when the input is larger), `img_ref` the Ref PIL-bicubic
    resized to gt_size x gt_size, both flipped / rotated alike, then x1/4 and x4 as in the test phase."""
    from PIL import Image
    if gt_size % scale:
        raise ValueError(f'gt_size {gt_size} is not a multiple of the scale {scale}')
    h, w = img_in.shape[:2]
    if h < gt_size or w < gt_size:
        raise ValueError(f'input {h}x{w} is smaller than gt_size {gt_size}: {path}')
    if (h, w) != (gt_size, gt_size):
        top, left = random.randint(0, h - gt_size), random.randint(0, w - gt_size)
        img_in = img_in[top:top + gt_size, left:left + gt_size]
    img_ref = _pil_to_bgr(_pil_resize_bgr(img_ref, (gt_size, gt_size)))
    img_in, img_ref = augment([img_in, img_ref], use_flip, use_rot)
    deg = _degraded(img_in, img_ref, scale)
    return {'img_in': _to_tensor_rgb(img_in), 'img_in_lq': deg['img_in_lq'], 'img_in_up': deg['img_in_up'],
            'img_ref': _to_tensor_rgb(img_ref), 'img_ref_lq': deg['img_ref_lq'], 'img_ref_up': deg['img_ref_up']}


def _paired_paths(opt):
    """(input, ref) path pairs: from `ann_file` ("<input> <ref>" per line, data/util.py:153-191) or, without one,
    every file of `dataroot_ref` paired with the input file of the same name (data/util.py:194-231)."""
    if opt.get('ann_file'):
        paths = []
        with open(opt['ann_file']) as f:
            for line in f:
                if line.strip():
                    a, b = line.strip().split(' ')
                    paths.append((osp.join(opt['dataroot_in'], a), osp.join(opt['dataroot_ref'], b)))
        return paths
    tmpl = opt.get('filename_tmpl') or '{}'
    ins, refs = sorted(os.listdir(opt['dataroot_in'])), sorted(os.listdir(opt['dataroot_ref']))
    if len(ins) != len(refs):
        raise ValueError(f'input and ref folders hold {len(ins)} and {len(refs)} images')
    paths = []
    for r in refs:
        base, ext = osp.splitext(r)
        name = tmpl.format(base) + ext
        if name not in ins:
            raise ValueError(f'{name} is not in {opt["dataroot_in"]}')
        paths.append((osp.join(opt['dataroot_in'], name), osp.join(opt['dataroot_ref'], r)))
    return paths


class RefCUFEDDataset(data.Dataset):

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        if (opt.get('io_backend') or {'type': 'disk'}).get('type', 'disk') != 'disk':
            raise NotImplementedError('only the disk io_backend is supported in the H100 build')
        self.train = opt.get('phase', 'test') == 'train'
        if self.train:
            self.paths = _paired_paths(opt)
        else:
            self.paths = []
            with open(opt['ann_file']) as f:       # "<input> <ref>" per line (data/util.py:153-191)
                for line in f:
                    a, b = line.strip().split(' ')
                    self.paths.append((osp.join(opt['dataroot_in'], a), osp.join(opt['dataroot_ref'], b)))

    def __len__(self):
        return len(self.paths)

    def pair_shape(self, i):
        """(padded H, padded W, GT h, GT w) of pair i from the image headers only — the batch bucketing key: every
        tensor of the sample dict has a shape determined by it (`img_in` is the UN-padded ground truth)."""
        from PIL import Image
        s = self.opt['scale']
        dims = []
        for p in self.paths[i]:
            with Image.open(p) as im:
                w, h = im.size
            dims.append((h - h % s, w - w % s))
        return (max(dims[0][0], dims[1][0]), max(dims[0][1], dims[1][1])) + dims[0]

    def __getitem__(self, i):
        import cv2
        in_path, ref_path = self.paths[i]
        rd = lambda p: cv2.imread(p, cv2.IMREAD_COLOR).astype(np.float32) / 255.0
        if self.train:
            return make_train_sample(rd(in_path), rd(ref_path), int(self.opt['gt_size']), self.opt['scale'],
                                     bool(self.opt.get('use_flip')), bool(self.opt.get('use_rot')), in_path)
        return make_sample(rd(in_path), rd(ref_path), self.opt['scale'], ref_path)


class SyntheticRefDataset(data.Dataset):
    """Seeded random pairs with CUFED5-like shapes: `num` pairs, `gt_size` HR input, `ref_size` Ref
    (BASELINE.json config 5: 126 pairs, 640x640 / 500x500).  In the train phase pair i is an `in_size` input
    (default gt_size, as CUFED's 160x160 training inputs) and a `ref_size` Ref through `make_train_sample`."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.num = int(opt.get('num', 126))
        self.gt = int(opt.get('gt_size', 640))
        self.ref = int(opt.get('ref_size', 500))

    def __len__(self):
        return self.num

    def pair_shape(self, i):
        s = self.opt.get('scale', 4)
        g = self.gt - self.gt % s
        m = max(g, self.ref - self.ref % s)
        return m, m, g, g

    def __getitem__(self, i):
        rng = np.random.default_rng(1234 + i)
        smooth = lambda n: np.clip(np.kron(rng.random((n // 8 + 1, n // 8 + 1, 3)), np.ones((8, 8, 1)))[:n, :n] * 0.7 +
                                   rng.random((n, n, 3)) * 0.3, 0, 1).astype(np.float32)
        if self.opt.get('phase', 'test') == 'train':
            img_in = smooth(int(self.opt.get('in_size') or self.gt))
            return make_train_sample(img_in, smooth(self.ref), self.gt, self.opt.get('scale', 4),
                                     bool(self.opt.get('use_flip')), bool(self.opt.get('use_rot')),
                                     f'synthetic_{i:04d}.png')
        return make_sample(smooth(self.gt), smooth(self.ref), self.opt.get('scale', 4), f'synthetic_{i:04d}.png')
