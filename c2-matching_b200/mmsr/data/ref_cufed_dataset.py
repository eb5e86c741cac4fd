"""Test-phase `RefCUFEDDataset` (reference: mmsr/data/ref_cufed_dataset.py:13-170) plus a
file-free synthetic stand-in with the same sample dict.

Per pair: mod-crop both images to the scale, zero-pad both (bottom/right) to a common size
(:99-114), PIL-bicubic x1/4 then x4 (:119-134), BGR->RGB CHW float tensors (:145-166)."""
import os.path as osp

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


def make_sample(img_in, img_ref, scale, path=''):
    """img_in / img_ref: float32 BGR HWC in [0,1] -> the reference's test-phase sample dict."""
    img_in, img_ref = _mod_crop(img_in, scale), _mod_crop(img_ref, scale)
    img_in_gt = img_in.copy()
    (ih, iw), (rh, rw) = img_in.shape[:2], img_ref.shape[:2]
    padding = (ih, iw) != (rh, rw)
    if padding:
        th, tw = max(ih, rh), max(iw, rw)
        img_in, img_ref = _pad_to(img_in, th, tw), _pad_to(img_ref, th, tw)
    gh, gw = img_in.shape[:2]
    lq = (gw // scale, gh // scale)
    bgr = lambda pil: np.asarray(pil)[..., ::-1].astype(np.float32) / 255.0
    in_lq = _pil_resize_bgr(img_in, lq)
    ref_lq = _pil_resize_bgr(img_ref, lq)
    from PIL import Image
    in_up, ref_up = in_lq.resize((gw, gh), Image.BICUBIC), ref_lq.resize((gw, gh), Image.BICUBIC)
    return {'img_in': _to_tensor_rgb(img_in_gt), 'img_in_lq': _to_tensor_rgb(bgr(in_lq)),
            'img_in_up': _to_tensor_rgb(bgr(in_up)), 'img_ref': _to_tensor_rgb(img_ref),
            'img_ref_lq': _to_tensor_rgb(bgr(ref_lq)), 'img_ref_up': _to_tensor_rgb(bgr(ref_up)),
            'lq_path': path, 'padding': padding, 'original_size': (ih, iw)}


class RefCUFEDDataset(data.Dataset):

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        if (opt.get('io_backend') or {'type': 'disk'}).get('type', 'disk') != 'disk':
            raise NotImplementedError('only the disk io_backend is supported in the H100 build')
        if opt.get('phase', 'test') == 'train':
            raise NotImplementedError('training datasets are outside the H100 hot-path scope')
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
        return make_sample(rd(in_path), rd(ref_path), self.opt['scale'], ref_path)


class SyntheticRefDataset(data.Dataset):
    """Seeded random pairs with CUFED5-like shapes: `num` pairs, `gt_size` HR input, `ref_size` Ref
    (BASELINE.json config 5: 126 pairs, 640x640 / 500x500)."""

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
        return make_sample(smooth(self.gt), smooth(self.ref), self.opt.get('scale', 4), f'synthetic_{i:04d}.png')
