"""Minimal stand-ins for the mmcv pieces the hot-path modules are built with.

The reference builds every attention module from a config dict through mmcv's registry
(`@ATTENTION.register_module()`, `build_attention(cfg)`; e.g.
projects/mmdet3d_plugin/bevformer/modules/spatial_cross_attention.py:29,61 and
projects/configs/vidar_pretrain/nusc_1_8_subset/vidar_1_8_nusc_3future.py:146-157).  mmcv is
not a dependency of this package, so the same contract is provided here: a name -> class
registry, `build_from_cfg`-style construction from `dict(type='Name', **kwargs)`, and the
few init helpers the modules call.  When a real mmcv is importable the modules are ALSO
registered into mmcv's own `ATTENTION` registry (see `register_into_mmcv`), which is what makes
them drop into an unchanged ViDAR config.
"""
import copy

import torch.nn as nn


class Registry:
    def __init__(self, name):
        self.name = name
        self._modules = {}

    def __contains__(self, key):
        return key in self._modules

    def get(self, key):
        return self._modules.get(key)

    @property
    def module_dict(self):
        return dict(self._modules)

    def register_module(self, name=None, force=False, module=None):
        def _register(cls):
            key = name or cls.__name__
            if key in self._modules and not force:
                raise KeyError(f"{key} is already registered in {self.name}")
            self._modules[key] = cls
            return cls
        if module is not None:
            return _register(module)
        return _register

    def build(self, cfg, default_args=None):
        return build_from_cfg(cfg, self, default_args)


def build_from_cfg(cfg, registry, default_args=None):
    if not isinstance(cfg, dict):
        raise TypeError(f"cfg must be a dict, but got {type(cfg)}")
    if "type" not in cfg and not (default_args and "type" in default_args):
        raise KeyError(f'`cfg` or `default_args` must contain the key "type", but got {cfg}')
    args = copy.deepcopy(cfg)
    if default_args:
        for k, v in default_args.items():
            args.setdefault(k, v)
    obj_type = args.pop("type")
    if isinstance(obj_type, str):
        cls = registry.get(obj_type)
        if cls is None:
            raise KeyError(f"{obj_type} is not in the {registry.name} registry")
    elif isinstance(obj_type, type):
        cls = obj_type
    else:
        raise TypeError(f"type must be a str or valid type, but got {type(obj_type)}")
    return cls(**args)


ATTENTION = Registry("attention")
TRANSFORMER_LAYER = Registry("transformerLayer")
TRANSFORMER_LAYER_SEQUENCE = Registry("transformer-layers sequence")


CONV_LAYERS = Registry("conv layer")
CONV_LAYERS.register_module("Conv2d", module=nn.Conv2d)
CONV_LAYERS.register_module("Conv", module=nn.Conv2d)


def build_attention(cfg, default_args=None):
    """mmcv.cnn.bricks.transformer.build_attention."""
    return build_from_cfg(cfg, ATTENTION, default_args)


def build_conv_layer(cfg, *args, **kwargs):
    """mmcv.cnn.build_conv_layer: `cfg` None means Conv2d; otherwise CONV_LAYERS[cfg['type']](*args, **kwargs, **rest of
    cfg), e.g. mmdet's ResNet `build_conv_layer(dict(type='DCNv2', deform_groups=1), planes, planes, kernel_size=3,
    stride=1, padding=1, dilation=1, bias=False)`."""
    from . import dcn  # noqa: F401  (registers DCNv2)
    cfg_ = dict(type="Conv2d") if cfg is None else copy.deepcopy(cfg)
    if not isinstance(cfg_, dict) or "type" not in cfg_:
        raise TypeError(f"cfg must be a dict with the key \"type\", but got {cfg}")
    layer_type = cfg_.pop("type")
    cls = CONV_LAYERS.get(layer_type)
    if cls is None:
        raise KeyError(f"Unrecognized conv type {layer_type}")
    return cls(*args, **kwargs, **cfg_)


class BaseModule(nn.Module):
    """mmcv.runner.base_module.BaseModule: nn.Module that remembers `init_cfg`."""

    def __init__(self, init_cfg=None):
        super().__init__()
        self._is_init = False
        self.init_cfg = copy.deepcopy(init_cfg)

    def init_weights(self):
        self._is_init = True


def constant_init(module, val, bias=0):
    if hasattr(module, "weight") and module.weight is not None:
        nn.init.constant_(module.weight, val)
    if hasattr(module, "bias") and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def xavier_init(module, gain=1, bias=0, distribution="normal"):
    assert distribution in ("uniform", "normal")
    if hasattr(module, "weight") and module.weight is not None:
        if distribution == "uniform":
            nn.init.xavier_uniform_(module.weight, gain=gain)
        else:
            nn.init.xavier_normal_(module.weight, gain=gain)
    if hasattr(module, "bias") and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def register_into_mmcv():
    """If mmcv is installed, expose this package's modules under the reference's names in
    mmcv's own ATTENTION registry (force=True replaces the plugin's classes), and its
    deformable convolution as `DCNv2` in mmcv's CONV_LAYERS (what mmdet's ResNet builds for
    `dcn=dict(type='DCNv2', ...)`), and its optimizer as `VidarAdamW` in mmcv's OPTIMIZERS (what `build_optimizer`
    builds for `optimizer=dict(type='VidarAdamW', ...)`)."""
    try:
        from mmcv.cnn.bricks.registry import ATTENTION as MMCV_ATTENTION
        from mmcv.cnn.bricks.registry import CONV_LAYERS as MMCV_CONV_LAYERS
        from mmcv.runner.optimizer import OPTIMIZERS as MMCV_OPTIMIZERS
    except Exception:
        return False
    from . import dcn  # noqa: F401  (registers DCNv2)
    from .optim import AdamW
    for name, cls in ATTENTION.module_dict.items():
        MMCV_ATTENTION.register_module(name=name, force=True, module=cls)
    for name, cls in CONV_LAYERS.module_dict.items():
        if cls.__module__.startswith(__package__ + "."):           # this package's ops only, not torch's Conv2d
            MMCV_CONV_LAYERS.register_module(name=name, force=True, module=cls)
    MMCV_OPTIMIZERS.register_module(name="VidarAdamW", force=True, module=AdamW)
    return True
