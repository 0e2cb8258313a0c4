"""HEADS / LOSSES / ROI_EXTRACTORS registries and build_from_cfg.

Mirrors mmdet/utils/registry.py:6-76, mmdet/models/registry.py:7-8 and
mmdet/models/builder.py:34-35 so that ``bbox_head=dict(type='GSBBoxHeadWith0', ...)``
blocks from configs/bags/*.py construct unchanged.  When a real mmdetection
(v1.x) is importable its own registries are used instead, which makes the head
a drop-in inside an existing mmdet installation (see INTEGRATION.md).
"""
from __future__ import annotations

import inspect


class Registry(object):

    def __init__(self, name):
        self._name = name
        self._module_dict = dict()

    def __repr__(self):
        return '{}(name={}, items={})'.format(self.__class__.__name__, self._name,
                                              list(self._module_dict.keys()))

    @property
    def name(self):
        return self._name

    @property
    def module_dict(self):
        return self._module_dict

    def get(self, key):
        return self._module_dict.get(key, None)

    def _register_module(self, module_class, force=False):
        if not inspect.isclass(module_class):
            raise TypeError('module must be a class, but got {}'.format(type(module_class)))
        module_name = module_class.__name__
        if module_name in self._module_dict and not force:
            raise KeyError('{} is already registered in {}'.format(module_name, self.name))
        self._module_dict[module_name] = module_class

    def register_module(self, cls=None, force=False):
        if cls is None:
            return lambda c: self.register_module(c, force=force)
        self._register_module(cls, force=force)
        return cls


def build_from_cfg(cfg, registry, default_args=None):
    """Same contract as mmdet/utils/registry.py:48-76."""
    assert isinstance(cfg, dict) and 'type' in cfg
    assert isinstance(default_args, dict) or default_args is None
    args = dict(cfg)
    obj_type = args.pop('type')
    if isinstance(obj_type, str):
        obj_cls = registry.get(obj_type)
        if obj_cls is None:
            raise KeyError('{} is not in the {} registry'.format(obj_type, registry.name))
    elif inspect.isclass(obj_type):
        obj_cls = obj_type
    else:
        raise TypeError('type must be a str or valid type, but got {}'.format(type(obj_type)))
    if default_args is not None:
        for name, value in default_args.items():
            args.setdefault(name, value)
    return obj_cls(**args)


def _mmdet_registries():
    try:  # pragma: no cover - mmdet is not installable in the build image
        from mmdet.models.registry import HEADS as _H, LOSSES as _L
        return _H, _L
    except Exception:
        return None


_ext = _mmdet_registries()
if _ext is not None:  # pragma: no cover
    HEADS, LOSSES = _ext
    USING_MMDET_REGISTRY = True
else:
    HEADS = Registry('head')
    LOSSES = Registry('loss')
    USING_MMDET_REGISTRY = False


def _mmdet_roi_extractors():
    try:  # pragma: no cover - mmdet is not installable in the build image
        from mmdet.models.registry import ROI_EXTRACTORS as _R
        return _R
    except Exception:
        return None


ROI_EXTRACTORS = _mmdet_roi_extractors()
if ROI_EXTRACTORS is None:
    ROI_EXTRACTORS = Registry('roi_extractor')


def build_head(cfg):
    return build_from_cfg(cfg, HEADS)


def build_loss(cfg):
    return build_from_cfg(cfg, LOSSES)


def build_roi_extractor(cfg):
    return build_from_cfg(cfg, ROI_EXTRACTORS)


def register(registry, cls):
    """register_module that tolerates both registry flavours and re-imports."""
    if registry.get(cls.__name__) is None:
        try:
            registry.register_module(cls)
        except TypeError:  # pragma: no cover - newer mmcv style
            registry.register_module()(cls)
    return cls
