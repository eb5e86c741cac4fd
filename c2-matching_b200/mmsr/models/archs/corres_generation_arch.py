"""Correspondence generation: dense LR<->Ref patch matching -> pre-offsets for the three DCN
scales, plus VGG19 Ref features (mmsr/models/archs/corres_generation_arch.py:14-117).

H100 path: ONE batched call normalises both feature maps per pixel, runs the fused
tensor-core (wgmma) correlation + argmax and the exact rescoring (csrc/corr_*.cu); the reference's Python
loop over the batch, the 230 MB patch copy and the 2 x 2.09 GB score tensors per image are gone.
The 9-shift x 3-scale offset pyramid is one small kernel per scale, produced lazily: the H100
RestorationNet consumes the index map directly and never needs it in HBM."""
import torch
from torch import nn

from c2m_b200 import ops as _ops

from .vgg_arch import VGGFeatureExtractor

_SCALES = {'relu3_1': 1, 'relu2_1': 2, 'relu1_1': 4}


class ScaleOffsets:
    """Handle for one pyramid level: index map + how to decode it."""
    __slots__ = ('max_idx', 'scale', 'ref_gw')

    def __init__(self, max_idx, scale, ref_gw):
        self.max_idx, self.scale, self.ref_gw = max_idx, scale, ref_gw

    def materialize(self):
        return _ops.offset_pyramid(self.max_idx, self.scale, self.ref_gw)


class PreOffsets(dict):
    """dict{'relu1_1','relu2_1','relu3_1' -> [B,9,H,W,2] (x,y) offsets} as the reference returns
    (corres_generation_arch.py:107-114), filled on first access; `.handle(k)` gives the fused path."""

    def __init__(self, max_idx, ref_gw):
        super().__init__()
        self.max_idx, self.ref_gw = max_idx, ref_gw

    def handle(self, key):
        return ScaleOffsets(self.max_idx, _SCALES[key], self.ref_gw)

    def __missing__(self, key):
        if key not in _SCALES:
            raise KeyError(key)
        t = self.handle(key).materialize()
        self[key] = t
        return t

    def _fill(self):
        for k in _SCALES:
            self[k]  # noqa: B018 — triggers __missing__
        return self

    def keys(self):
        return dict.keys(self._fill())

    def items(self):
        return dict.items(self._fill())

    def values(self):
        return dict.values(self._fill())

    def __iter__(self):
        return dict.__iter__(self._fill())

    def __contains__(self, key):
        return key in _SCALES

    def get(self, key, default=None):
        return self[key] if key in _SCALES else default

    def __len__(self):
        return len(_SCALES)


class CorrespondenceGenerationArch(nn.Module):

    def __init__(self, patch_size=3, stride=1, vgg_layer_list=('relu3_1', 'relu2_1', 'relu1_1'),
                 vgg_type='vgg19', vgg_pretrained=None, vgg_pretrained_path=None):
        """Reference signature (corres_generation_arch.py:16-27) + two optional kwargs: the reference builds
        `vgg19(pretrained=True)` here and never loads net_map from a checkpoint, so by default the ImageNet
        weights are REQUIRED (local checkpoint or torch hub cache; raises otherwise)."""
        super().__init__()
        self.patch_size, self.stride = patch_size, stride
        self.vgg_layer_list = list(vgg_layer_list)
        self.vgg = VGGFeatureExtractor(layer_name_list=self.vgg_layer_list, vgg_type=vgg_type,
                                       pretrained=vgg_pretrained, pretrained_path=vgg_pretrained_path)

    def index_to_flow(self, max_idx):
        """[h,w] index map -> [1,h+2,w+2,2] (x,y) flow, zero-padded (corres…:29-46)."""
        return _ops.offset_pyramid(max_idx.unsqueeze(0), 1)[:, 0]

    def match(self, dense_features):
        f_in, f_ref = dense_features['dense_features1'], dense_features['dense_features2']
        if f_in.shape != f_ref.shape:
            # the reference views feat_ref with feat_in's (c,h,w) (:55-58): equal sizes are required
            raise RuntimeError(f'input/Ref feature maps differ: {tuple(f_in.shape)} vs {tuple(f_ref.shape)}')
        idx, _ = _ops.corr_argmax(f_in, f_ref, self.patch_size, self.stride, self.stride, is_norm=True,
                                  norm_input=True, l2norm=True)
        return idx

    def forward(self, dense_features, img_ref_hr):
        idx = self.match(dense_features)
        pre_offset = PreOffsets(idx, idx.shape[2])     # decode width = INPUT grid width (:32-34)
        img_ref_feat = self.vgg(img_ref_hr, packed=True)     # dict of fp32 features, materialised lazily
        return pre_offset, img_ref_feat
