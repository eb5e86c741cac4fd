"""Options-YAML API (reference: mmsr/utils/options.py): `parse`, `dict2str`, `NoneDict`,
`dict_to_nonedict`.  Reference option files (options/test/*.yml) are accepted verbatim."""
import os
import os.path as osp
from collections import OrderedDict

import yaml


def ordered_yaml():
    """yaml Loader/Dumper pair that keeps mapping order (options.py:8-29)."""
    try:
        from yaml import CDumper as Dumper, CLoader as Loader
    except ImportError:
        from yaml import Dumper, Loader
    tag = yaml.resolver.BaseResolver.DEFAULT_MAPPING_TAG
    Dumper.add_representer(OrderedDict, lambda dumper, data: dumper.represent_dict(data.items()))
    Loader.add_constructor(tag, lambda loader, node: OrderedDict(loader.construct_pairs(node)))
    return Loader, Dumper


def parse(opt_path, is_train=True):
    """YAML file -> option dict with the derived keys of options.py:32-98."""
    with open(opt_path) as f:
        opt = yaml.load(f, Loader=ordered_yaml()[0])
    gpu_ids = opt.get('gpu_ids') or []
    gpu_list = ','.join(str(x) for x in gpu_ids)
    if opt.get('set_CUDA_VISIBLE_DEVICES'):
        os.environ['CUDA_VISIBLE_DEVICES'] = gpu_list
        print('export CUDA_VISIBLE_DEVICES=' + gpu_list, flush=True)
    else:
        print('gpu_list: ', gpu_list, flush=True)
    opt['is_train'] = is_train
    scale = opt['scale']
    if opt.get('crop_border') is None:
        opt['crop_border'] = scale
    for phase, dataset in (opt.get('datasets') or {}).items():
        dataset['phase'] = phase.split('_')[0]
        dataset['scale'] = scale
        for k in ('dataroot_gt', 'dataroot_lq'):
            if dataset.get(k) is not None:
                dataset[k] = osp.expanduser(dataset[k])
    opt.setdefault('path', OrderedDict())
    for key, path in list(opt['path'].items()):
        if path and key != 'strict_load':
            opt['path'][key] = osp.expanduser(path)
    root = osp.abspath(osp.join(osp.dirname(osp.abspath(__file__)), osp.pardir, osp.pardir))
    opt['path']['root'] = root
    if is_train:
        # `path.experiments_root` in the file moves a run's directory out of the package tree
        exp = opt['path'].get('experiments_root') or osp.join(root, 'experiments', opt['name'])
        opt['path'].update(experiments_root=exp, models=osp.join(exp, 'models'),
                           training_state=osp.join(exp, 'training_state'), log=exp,
                           visualization=osp.join(exp, 'visualization'))
    else:
        res = osp.join(root, 'results', opt['name'])
        opt['path'].update(results_root=res, log=res, visualization=osp.join(res, 'visualization'))
    return opt


def dict2str(opt, indent_level=1):
    pad = ' ' * (indent_level * 2)
    msg = ''
    for k, v in opt.items():
        if isinstance(v, dict):
            msg += f'{pad}{k}:[\n{dict2str(v, indent_level + 1)}{pad}]\n'
        else:
            msg += f'{pad}{k}: {v}\n'
    return msg


class NoneDict(dict):
    """Missing keys read as None (options.py:122-126)."""

    def __missing__(self, key):
        return None


def dict_to_nonedict(opt):
    if isinstance(opt, dict):
        return NoneDict(**{k: dict_to_nonedict(v) for k, v in opt.items()})
    if isinstance(opt, list):
        return [dict_to_nonedict(v) for v in opt]
    return opt
