"""VGG trunks with the reference's layer names (mmsr/models/archs/vgg_arch.py:7-145).

Built layer by layer here (no torchvision model object, no download at construction): only
the convolutions up to the deepest requested layer exist, exactly like the reference's
`features[:max_idx + 1]` slice, so state-dict keys are `vgg_net.conv{b}_{i}.{weight,bias}` plus
the `mean` / `std` buffers.  ImageNet weights, when wanted, are loaded with `load_imagenet()`
from a local torchvision checkpoint (the reference downloads them in the constructor)."""
from collections import OrderedDict

import torch
from torch import nn

_CFG = {  # convs per block
    'vgg11': (1, 1, 2, 2, 2), 'vgg13': (2, 2, 2, 2, 2), 'vgg16': (2, 2, 3, 3, 3), 'vgg19': (2, 2, 4, 4, 4),
}
_WIDTH = (64, 128, 256, 512, 512)


def layer_names(vgg_type):
    """['conv1_1','relu1_1',...,'pool5'] — vgg_arch.py:7-41 NAMES."""
    names = []
    for b, n in enumerate(_CFG[vgg_type.replace('_bn', '')], start=1):
        for i in range(1, n + 1):
            names += [f'conv{b}_{i}', f'relu{b}_{i}']
        names.append(f'pool{b}')
    return names


NAMES = {k: layer_names(k) for k in _CFG}


def build_trunk(vgg_type, last_layer, pooling_stride=2, remove_pooling=False):
    """Sequential of named layers up to and including `last_layer`."""
    seq = OrderedDict()
    cin = 3
    for name in layer_names(vgg_type):
        if name.startswith('conv'):
            cout = _WIDTH[int(name[4]) - 1]
            seq[name] = nn.Conv2d(cin, cout, 3, 1, 1)
            cin = cout
        elif name.startswith('relu'):
            seq[name] = nn.ReLU(inplace=True)
        elif not remove_pooling:
            seq[name] = nn.MaxPool2d(kernel_size=2, stride=pooling_stride)
        if name == last_layer:
            break
    else:
        raise ValueError(f'{last_layer} is not a layer of {vgg_type}')
    return nn.Sequential(seq)


_TV_FILES = {'vgg11': 'vgg11-8a719046.pth', 'vgg13': 'vgg13-19584684.pth', 'vgg16': 'vgg16-397923af.pth',
             'vgg19': 'vgg19-dcbb9e9d.pth'}


def find_imagenet_checkpoint(vgg_type, path=None):
    """Where the torchvision ImageNet checkpoint of `vgg_type` is on this machine, or None:
    explicit path -> $C2M_<VGG_TYPE>_WEIGHTS -> the torch hub cache torchvision downloads into."""
    import os
    cands = [path, os.environ.get(f'C2M_{vgg_type.upper()}_WEIGHTS')]
    try:
        cands.append(os.path.join(torch.hub.get_dir(), 'checkpoints', _TV_FILES[vgg_type]))
    except Exception:
        pass
    for c in cands:
        if c and os.path.isfile(c):
            return c
    return None


def load_imagenet(trunk, vgg_type, path=None):
    """Copy torchvision ImageNet weights (`features.N.*`) into a named trunk — what the reference's
    constructor does with `vgg19(pretrained=True)` (vgg_arch.py:103-104).  Resolution: `path`,
    $C2M_VGG19_WEIGHTS, the torch hub cache, then torchvision's own download.  Raises when none of them
    yields weights: a net_map with random VGG weights gives silently wrong SR images."""
    found = find_imagenet_checkpoint(vgg_type, path)
    if path is not None and found != path:
        raise FileNotFoundError(f'VGG checkpoint {path} not found')
    if found is not None:
        tv = torch.load(found, map_location='cpu')
    else:
        try:
            import torchvision
            tv = getattr(torchvision.models, vgg_type)(weights='IMAGENET1K_V1').state_dict()
        except Exception as e:
            raise RuntimeError(
                f'ImageNet weights for {vgg_type} are not available (no local checkpoint, download failed: {e}). '
                f'Put torchvision\'s {_TV_FILES.get(vgg_type)} into the torch hub cache, point '
                f'$C2M_{vgg_type.upper()}_WEIGHTS / the `vgg_pretrained_path` option at it, or pass vgg_pretrained=False '
                f'(C2M_VGG_PRETRAINED=0) if random VGG weights are intended (synthetic benchmarks).') from e
    convs = [m for m in trunk if isinstance(m, nn.Conv2d)]
    keys = sorted({int(k.split('.')[1]) for k in tv if k.startswith('features.')})
    with torch.no_grad():      # in-place copy_ on the parameter bumps its version -> packed-weight caches refresh
        for m, n in zip(convs, keys):
            m.weight.copy_(tv[f'features.{n}.weight'])
            m.bias.copy_(tv[f'features.{n}.bias'])


def pretrained_default():
    """The reference always builds its VGGs with pretrained=True; C2M_VGG_PRETRAINED=0 (set by the
    synthetic tests / bench, which have no ImageNet checkpoint) turns that off process-wide."""
    import os
    return os.environ.get('C2M_VGG_PRETRAINED', '1') != '0'


class PackedFeatures(dict):
    """{layer_name: fp32 feature} as the reference's extractor returns (vgg_arch.py:136-145), but the
    features live in the packed-split operand layout the tensor-core kernels consume (`.psa(name)`); the
    fp32 tensor of a layer is produced on first access only (none is, on the fused inference path)."""

    def __init__(self, packed):
        super().__init__()
        self._packed = dict(packed)

    def psa(self, key):
        return self._packed[key]

    def __missing__(self, key):
        from . import arch_util
        from c2m_b200 import ops
        if key not in self._packed:
            raise KeyError(key)
        t = arch_util.attach_psa(ops.psa_to_f32(self._packed[key]), self._packed[key])
        self[key] = t
        return t

    def _fill(self):
        for k in self._packed:
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
        return key in self._packed

    def get(self, key, default=None):
        return self[key] if key in self._packed else default

    def __len__(self):
        return len(self._packed)


def run_trunk(trunk, x, taps=(), want_last_f32=True, packed_taps=False):
    """Run a named VGG trunk (Sequential of conv / relu / pool).  Returns (last, {tap: fp32}), or
    (last, PackedFeatures) with packed_taps when the tensor-core path runs.

    tensor-core path: each conv+ReLU pair is one launch in the packed-split layout; a tapped ReLU
    output is written both as fp32 (for the DCN sampler / the caller) and packed (attached to the
    fp32 tensor for the next consumer); convs before a max-pool emit fp32 for torch's pooling."""
    from . import arch_util
    from c2m_b200 import ops
    layers = list(trunk.named_children())
    convs = [m for _, m in layers if isinstance(m, nn.Conv2d)]
    if not arch_util.psa_path_ok(x, *convs) or x.shape[2] < 72 or x.shape[3] < 40:
        got = {}
        for name, layer in layers:
            if isinstance(layer, nn.ReLU):
                x = torch.relu(x)
            else:
                x = layer(x)
            if name in taps:
                got[name] = x
        return x, got
    got = {}
    # PSA scale exponents of the trunk's INTERNAL activations (tapped outputs stay at 0: their consumers — the DCN
    # gather and the two-input convolutions — take exponent 0).  Calibrated on the first call from the activations'
    # amax (one synchronising pass, then cached on the trunk), so that tensors with small magnitudes keep their lo
    # halves out of the fp16 subnormal range and large ones keep 16x headroom below 65504.
    sa_tab = getattr(trunk, '_c2m_sa', None)
    calibrating = sa_tab is None
    if calibrating:
        sa_tab = {}
    sa_in = sa_tab.get('__input__', 0)
    if calibrating:
        sa_in = sa_tab['__input__'] = ops.suggest_sa(float(x.abs().max()))
    xp, xf = ops.psa_from_f32(x, sa_in), None
    i = 0
    while i < len(layers):
        name, layer = layers[i]
        if isinstance(layer, nn.Conv2d):
            has_relu = i + 1 < len(layers) and isinstance(layers[i + 1][1], nn.ReLU)
            out_name = layers[i + 1][0] if has_relu else name
            nxt = layers[i + 2][1] if has_relu and i + 2 < len(layers) else (layers[i + 1][1] if not has_relu and i + 1 < len(layers) else None)
            last = nxt is None
            pool_next = isinstance(nxt, nn.MaxPool2d) and nxt.kernel_size in (2, (2, 2)) and nxt.stride in (2, (2, 2))
            need_f32 = (out_name in taps and not packed_taps) or (isinstance(nxt, nn.MaxPool2d) and not pool_next) or \
                (last and want_last_f32)
            need_psa = isinstance(nxt, nn.Conv2d) or out_name in taps or pool_next
            if xp is None:
                xp = ops.psa_from_f32(xf)
            # tapped features feed the DCN sampler, which gathers 8-channel octets: keep them channels-last
            sa_out = 0 if (out_name in taps or not need_psa) else sa_tab.get(out_name, 0)
            r = ops.conv3x3_psa(xp, layer.weight, layer.bias, act='relu' if has_relu else None, psa_out=need_psa,
                                out_f32=need_f32, channels_last=out_name in taps, sa_out=sa_out)
            if calibrating and need_psa and out_name not in taps:
                pr = r[0] if (need_psa and need_f32) else r
                sa_new = ops.suggest_sa(ops.psa_amax(pr))
                sa_tab[out_name] = sa_new
                if sa_new != 0:      # redo this layer at its calibrated exponent so the first call already uses it
                    r = ops.conv3x3_psa(xp, layer.weight, layer.bias, act='relu' if has_relu else None, psa_out=need_psa,
                                        out_f32=need_f32, channels_last=out_name in taps, sa_out=sa_new)
            if need_psa and need_f32:
                xp, xf = r
                arch_util.attach_psa(xf, xp)
            elif need_psa:
                xp, xf = r, None
            else:
                xp, xf = None, r
            if out_name in taps:
                got[out_name] = xp if packed_taps else xf
            i += 2 if has_relu else 1
        elif isinstance(layer, nn.MaxPool2d):
            if xp is not None and layer.kernel_size in (2, (2, 2)) and layer.stride in (2, (2, 2)):
                xp, xf = ops.psa_maxpool2(xp), None          # stays in the operand layout
            else:
                xf = layer(xf if xf is not None else ops.psa_to_f32(xp))
                xp = None
            i += 1
        else:
            raise RuntimeError(f'unexpected layer {name} in VGG trunk')
    if calibrating:
        try:
            trunk._c2m_sa = sa_tab
        except Exception:
            pass
    if xf is None and (want_last_f32 or not packed_taps):
        xf = ops.psa_to_f32(xp)
    return xf, (PackedFeatures(got) if packed_taps else got)


class VGGFeatureExtractor(nn.Module):
    """Returns {layer_name: feature} for the requested layers — vgg_arch.py:59-145."""

    def __init__(self, layer_name_list, vgg_type='vgg19', use_input_norm=True, requires_grad=False,
                 remove_pooling=False, pooling_stride=2, pretrained=None, pretrained_path=None):
        super().__init__()
        if 'bn' in vgg_type:
            raise NotImplementedError('batch-norm VGG variants are not used by C2-Matching')
        self.layer_name_list = list(layer_name_list)
        self.use_input_norm = use_input_norm
        self.names = layer_names(vgg_type)
        last = max(self.layer_name_list, key=self.names.index)
        self.vgg_net = build_trunk(vgg_type, last, pooling_stride, remove_pooling)
        # reference: `vgg19(pretrained=True)` in the constructor (vgg_arch.py:103-104); `pretrained=False`
        # / C2M_VGG_PRETRAINED=0 are this build's explicit opt-outs for synthetic weights
        if pretrained is None:
            pretrained = pretrained_default() or pretrained_path is not None
        if pretrained:
            load_imagenet(self.vgg_net, vgg_type, pretrained_path)
        if not requires_grad:
            for p in self.parameters():
                p.requires_grad = False
        if use_input_norm:
            self.register_buffer('mean', torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
            self.register_buffer('std', torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))

    def forward(self, x, packed=False):
        """packed=True (inference): features stay in the tensor-core operand layout, fp32 on demand."""
        if self.use_input_norm:
            x = (x - self.mean) / self.std
        _, got = run_trunk(self.vgg_net, x, taps=self.layer_name_list, want_last_f32=False,
                           packed_taps=packed and not torch.is_grad_enabled())
        return got
