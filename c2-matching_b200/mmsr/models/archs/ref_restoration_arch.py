"""Restoration generator (mmsr/models/archs/ref_restoration_arch.py:8-187): LR content features,
then three scales of [offset convs -> dynamic aggregation (DCN over Ref features) -> head ->
16 ResBlocks -> upsample], plus a bilinear x4 skip.

Same constructor (`ngf, n_blocks, groups`) and state-dict keys as the reference, so
`c2_matching_restoration_*.pth` loads with strict=True.  Differences are execution only: each
dynamic-aggregation tail is one fused kernel (see DCNv2/dcn_v2.py) including its LeakyReLU, and
the pre-offsets are read straight from the index map when CorrespondenceGenerationArch
provides a PreOffsets handle."""
import torch
import torch.nn.functional as F
from torch import nn

from . import arch_util
from .DCNv2.dcn_v2 import DCN_sep_pre_multi_offset as DynAgg

_LEVELS = (('small', 'relu3_1', 256), ('medium', 'relu2_1', 128), ('large', 'relu1_1', 64))


class ContentExtractor(nn.Module):

    def __init__(self, in_nc=3, out_nc=3, nf=64, n_blocks=16):
        super().__init__()
        self.conv_first = arch_util.Conv2d(in_nc, nf, 3, 1, 1)
        self.body = arch_util.make_layer(arch_util.ResidualBlockNoBN, n_blocks, nf=nf)
        arch_util.default_init_weights([self.conv_first], 0.1)

    def forward_psa(self, x):
        from c2m_b200 import ops
        hp = arch_util.conv_psa(self.conv_first, ops.psa_from_f32(x), act='lrelu')
        return arch_util.resblocks_psa(self.body, hp)

    def forward(self, x):
        from c2m_b200 import ops
        if arch_util.psa_path_ok(x, self.conv_first, self.body[0].conv1):
            return ops.psa_to_f32(self.forward_psa(x))
        return self.body(F.leaky_relu(self.conv_first(x), 0.1))


class DynamicAggregationRestoration(nn.Module):

    def __init__(self, ngf=64, n_blocks=16, groups=8):
        super().__init__()
        for size, _, c in _LEVELS:
            setattr(self, f'{size}_offset_conv1', arch_util.Conv2d(ngf + c, c, 3, 1, 1, bias=True))
            setattr(self, f'{size}_offset_conv2', arch_util.Conv2d(c, c, 3, 1, 1, bias=True))
            setattr(self, f'{size}_dyn_agg', DynAgg(c, c, 3, stride=1, padding=1, dilation=1,
                                                    deformable_groups=groups, extra_offset_mask=True))
            setattr(self, f'head_{size}', nn.Sequential(arch_util.Conv2d(ngf + c, ngf, 3, 1, 1), nn.LeakyReLU(0.1, True)))
            setattr(self, f'body_{size}', arch_util.make_layer(arch_util.ResidualBlockNoBN, n_blocks, nf=ngf))
        self.tail_small = nn.Sequential(arch_util.Conv2d(ngf, ngf * 4, 3, 1, 1), nn.PixelShuffle(2), nn.LeakyReLU(0.1, True))
        self.tail_medium = nn.Sequential(arch_util.Conv2d(ngf, ngf * 4, 3, 1, 1), nn.PixelShuffle(2), nn.LeakyReLU(0.1, True))
        self.tail_large = nn.Sequential(arch_util.Conv2d(ngf, ngf // 2, 3, 1, 1), nn.LeakyReLU(0.1, True),
                                        arch_util.Conv2d(ngf // 2, 3, 3, 1, 1))

    @staticmethod
    def _pre(pre_offset, key):
        return pre_offset.handle(key) if hasattr(pre_offset, 'handle') else pre_offset[key]

    def forward(self, x, pre_offset, img_ref_feat):
        """Module path: plain convolutions through cuDNN (used for tiny maps / C2M_FAST_CONV=0)."""
        for size, key, _ in _LEVELS:
            ref = img_ref_feat[key]
            off = torch.cat([x, ref], 1)
            off = F.leaky_relu_(getattr(self, f'{size}_offset_conv1')(off), 0.1)
            off = F.leaky_relu_(getattr(self, f'{size}_offset_conv2')(off), 0.1)
            swapped = getattr(self, f'{size}_dyn_agg')([ref, off], self._pre(pre_offset, key), lrelu_slope=0.1)
            h = getattr(self, f'head_{size}')(torch.cat([x, swapped], 1))
            h = arch_util.body_forward(getattr(self, f'body_{size}'), h, skip=x)
            x = getattr(self, f'tail_{size}')(h)
        return x

    def forward_psa(self, xp, pre_offset, img_ref_feat, base):
        """tensor-core path: every plain convolution runs in the packed-split layout; `cat` is a
        two-input convolution, PixelShuffle and the final `+ base` are conv epilogues; only the
        DCN boundary (fp32 offsets/mask in, fp32 features out) leaves the layout."""
        from c2m_b200 import ops
        out = None
        for size, key, _ in _LEVELS:
            if hasattr(img_ref_feat, 'psa'):
                ref = refp = img_ref_feat.psa(key)       # PackedFeatures: no fp32 copy of the Ref features
            else:
                ref = img_ref_feat[key]
                refp = arch_util.psa_of(ref)
            dyn = getattr(self, f'{size}_dyn_agg')
            off = arch_util.conv_psa(getattr(self, f'{size}_offset_conv1'), xp, act='lrelu', x2=refp)
            off = arch_util.conv_psa(getattr(self, f'{size}_offset_conv2'), off, act='lrelu')
            om = arch_util.conv_psa(dyn.conv_offset_mask, off, psa_out=False, out_f32=True, f32_octets=True)
            swapped = dyn.fused_tail(ref, om, self._pre(pre_offset, key), lrelu_slope=0.1, want_psa=True)
            h = arch_util.conv_psa(getattr(self, f'head_{size}')[0], xp, act='lrelu', x2=swapped)
            h = arch_util.resblocks_psa(getattr(self, f'body_{size}'), h, final_residual2=xp)
            tail = getattr(self, f'tail_{size}')
            if size != 'large':
                xp = arch_util.conv_psa(tail[0], h, act='lrelu', pixel_shuffle=2)
            else:
                t = arch_util.conv_psa(tail[0], h, act='lrelu')
                out = arch_util.conv_psa(tail[2], t, psa_out=False, out_f32=True, add_f32=base)
        return out


class RestorationNet(nn.Module):

    def __init__(self, ngf=64, n_blocks=16, groups=8):
        super().__init__()
        self.content_extractor = ContentExtractor(in_nc=3, out_nc=3, nf=ngf, n_blocks=n_blocks)
        self.dyn_agg_restore = DynamicAggregationRestoration(ngf, n_blocks, groups)
        arch_util.srntt_init_weights(self, init_type='normal', init_gain=0.02)
        self.re_init_dcn_offset()

    def re_init_dcn_offset(self):
        for size, _, _ in _LEVELS:
            getattr(self.dyn_agg_restore, f'{size}_dyn_agg').init_offset()

    def forward(self, x, pre_offset, img_ref_feat):
        base = F.interpolate(x, None, 4, 'bilinear', False)
        ce, dr = self.content_extractor, self.dyn_agg_restore
        # the offset / head convolutions consume cat[content (ngf channels), ref]: ngf must be a multiple of 32 for the
        # two-input tensor-core convolution, otherwise the module path below runs
        if arch_util.psa_path_ok(x, ce.conv_first, dr.small_offset_conv1, dr.head_small[0], dr.tail_large[2],
                                 cat_first=ce.conv_first.out_channels):
            return dr.forward_psa(ce.forward_psa(x), pre_offset, img_ref_feat, base.contiguous())
        content_feat = ce(x)
        return dr(content_feat, pre_offset, img_ref_feat) + base
