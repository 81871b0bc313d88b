"""Model registry and factory with the reference's surface (fastervit/models/registry.py:30-205):
`create_model(model_name, pretrained=False, checkpoint_path='', **kwargs)`, `list_models`, `is_model`,
`model_entrypoint`, `load_checkpoint`. Entrypoints are also offered to timm's registry when timm is
importable, so `timm.create_model('faster_vit_0_224')` (validate.py:195, train.py:428) resolves here.
"""
from __future__ import annotations

import fnmatch
import re
from collections import OrderedDict

import torch

from .configs import MODEL_SPECS, default_cfgs
from .model import build_model

_model_entrypoints: dict = {}


def _natural_key(s: str):
    return [int(p) if p.isdigit() else p for p in re.split(r"(\d+)", s.lower())]


def register_pip_model(fn):
    _model_entrypoints[fn.__name__] = fn
    return fn


def _make_entrypoint(name: str):
    def entry(pretrained=False, **kwargs):
        return build_model(name, pretrained=pretrained, **kwargs)
    entry.__name__ = entry.__qualname__ = name
    entry.__doc__ = f"FasterViT entrypoint `{name}` (H100-native); kwargs override {sorted(MODEL_SPECS[name]['defaults'])}."
    return entry


for _name in MODEL_SPECS:
    _fn = register_pip_model(_make_entrypoint(_name))
    globals()[_name] = _fn
    try:  # optional: make timm.create_model(name) work when timm is installed
        from timm.models import register_model as _timm_register  # type: ignore
        _fn.__module__ = __name__
        _timm_register(_fn)
    except Exception:
        pass


def list_models(filter: str = '', module: str = '', pretrained: bool = False, exclude_filters='',
                name_matches_cfg: bool = False):
    names = list(_model_entrypoints)
    if filter:
        names = fnmatch.filter(names, filter)
    if exclude_filters:
        ex = [exclude_filters] if isinstance(exclude_filters, str) else list(exclude_filters)
        for pat in ex:
            drop = set(fnmatch.filter(names, pat))
            names = [n for n in names if n not in drop]
    if pretrained:
        names = [n for n in names if 'http' in default_cfgs.get(n, {}).get('url', '')]
    return sorted(names, key=_natural_key)


def is_model(model_name: str) -> bool:
    return model_name in _model_entrypoints


def model_entrypoint(model_name: str):
    return _model_entrypoints[model_name]


def load_state_dict(checkpoint_path: str, use_ema: bool = False):
    """Read a checkpoint file and return its (EMA-)state_dict with any `module.` prefix removed
    (registry.py:161-186)."""
    ckpt = torch.load(checkpoint_path, map_location='cpu')
    key = ''
    if isinstance(ckpt, dict):
        if use_ema and 'state_dict_ema' in ckpt:
            key = 'state_dict_ema'
        elif 'state_dict' in ckpt:
            key = 'state_dict'
        elif 'model' in ckpt:
            key = 'model'
    sd = ckpt[key] if key else ckpt
    out = OrderedDict()
    for k, v in sd.items():
        out[k[7:] if k.startswith('module.') else k] = v
    if out and sorted(out)[0].startswith('encoder'):  # fv.py:206-207
        out = OrderedDict((k.replace('encoder.', ''), v) for k, v in out.items() if k.startswith('encoder.'))
    return out


def read_checkpoint_state(filename: str):
    """fv.py:172-209 (`_load_checkpoint`): `state_dict` / `model` / bare dict, `module.` prefix removed when the
    first key has it, `encoder.` sub-tree selected when the sorted-first key starts with `encoder`."""
    ckpt = torch.load(filename, map_location='cpu')
    if not isinstance(ckpt, dict):
        raise RuntimeError(f'No state_dict found in checkpoint file {filename}')
    sd = ckpt['state_dict'] if 'state_dict' in ckpt else (ckpt['model'] if 'model' in ckpt else ckpt)
    if list(sd.keys())[0].startswith('module.'):
        sd = {k[7:]: v for k, v in sd.items()}
    if sorted(sd.keys())[0].startswith('encoder'):
        sd = {k.replace('encoder.', ''): v for k, v in sd.items() if k.startswith('encoder.')}
    return sd


def load_state_dict_tolerant(module, state_dict, strict: bool = False, logger=None):
    """fv.py:112-168 (`_load_state_dict`): walk the module tree with `_load_from_state_dict` so that size
    mismatches are collected as messages (and those tensors left untouched) instead of raised; the summary is
    printed (or logged) unless `strict`, in which case it raises RuntimeError like the reference."""
    unexpected, all_missing, err_msg = [], [], []
    metadata = getattr(state_dict, '_metadata', None)
    state_dict = dict(state_dict) if not isinstance(state_dict, OrderedDict) else state_dict.copy()
    if metadata is not None:
        state_dict._metadata = metadata

    def load(mod, prefix=''):
        local = {} if metadata is None else metadata.get(prefix[:-1], {})
        mod._load_from_state_dict(state_dict, prefix, local, True, all_missing, unexpected, err_msg)
        for name, child in mod._modules.items():
            if child is not None:
                load(child, prefix + name + '.')

    load(module)
    missing = [k for k in all_missing if 'num_batches_tracked' not in k]
    if unexpected:
        err_msg.append('unexpected key in source ' f'state_dict: {", ".join(unexpected)}\n')
    if missing:
        err_msg.append(f'missing keys in source state_dict: {", ".join(missing)}\n')
    if err_msg:
        err_msg.insert(0, 'The model and loaded state dict do not match exactly\n')
        msg = '\n'.join(err_msg)
        if strict:
            raise RuntimeError(msg)
        if logger is not None:
            logger.warning(msg)
        else:
            print(msg)
    return missing, unexpected


def load_checkpoint(model, checkpoint_path: str, use_ema: bool = False, strict: bool = True):
    sd = load_state_dict(checkpoint_path, use_ema)
    return model.load_state_dict(sd, strict=strict)


def create_model(model_name: str, pretrained: bool = False, checkpoint_path: str = '', **kwargs):
    """registry.py:195-205."""
    if not is_model(model_name):
        raise RuntimeError('Unknown model (%s)' % model_name)
    model = model_entrypoint(model_name)(pretrained=pretrained, **kwargs)
    if checkpoint_path:
        load_checkpoint(model, checkpoint_path)
    return model
