"""Import the reference's pure-PyTorch modules in THIS container (no mmcv/mmdet installed).

Used only by the golden-vector generators under tools/ (test infrastructure).  It installs
throw-away stand-ins for the mmcv / mmdet / mmdet3d names the reference files import at
module level, and maps a synthetic package `vidar_ref` onto
/root/reference/projects/mmdet3d_plugin/bevformer so that files are loaded one by one
(relative imports work, the plugin's heavy __init__ chain is not executed).
`mmcv.ops.multi_scale_deform_attn.multi_scale_deformable_attn_pytorch` -- the reference's CPU
path for MSDA, whose source lives in the un-vendored mmcv-full 1.4.0 -- is provided by the
same-lineage implementation in `transformers` (NOT by this repo's oracle, so the goldens stay
independent of it).
"""
import importlib
import importlib.util
import os
import sys
import types

import torch
import torch.nn as nn

REF_BEVFORMER = "/root/reference/projects/mmdet3d_plugin/bevformer"


class _Anything:
    """Placeholder usable as decorator, base class factory, callable or namespace."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        if len(a) == 1 and callable(a[0]) and not k:
            return a[0]
        return _Anything()

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Anything()


class _Permissive(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Anything()


class _Registry:
    def __init__(self):
        self.modules = {}

    def register_module(self, name=None, force=False, module=None):
        def deco(cls):
            self.modules[name or cls.__name__] = cls
            return cls
        return deco(module) if module is not None else deco

    def build(self, cfg):
        cfg = dict(cfg)
        return self.modules[cfg.pop("type")](**cfg)


def _passthrough_decorator(*dargs, **dkw):
    if len(dargs) == 1 and callable(dargs[0]) and not dkw:
        return dargs[0]

    def deco(fn):
        return fn
    return deco


def _msda_pytorch(value, value_spatial_shapes, sampling_locations, attention_weights):
    from transformers.models.deformable_detr.modeling_deformable_detr import MultiScaleDeformableAttention
    shapes = [(int(h), int(w)) for h, w in value_spatial_shapes.tolist()]
    return MultiScaleDeformableAttention().forward(value, value_spatial_shapes, shapes, None,
                                                   sampling_locations, attention_weights, 64)


def install():
    if "vidar_ref" in sys.modules:
        return sys.modules["vidar_ref"]
    attention, layer, seq = _Registry(), _Registry(), _Registry()

    class BaseModule(nn.Module):
        def __init__(self, init_cfg=None):
            super().__init__()
            self.init_cfg = init_cfg

    def constant_init(m, val, bias=0):
        nn.init.constant_(m.weight, val)
        if m.bias is not None:
            nn.init.constant_(m.bias, bias)

    def xavier_init(m, gain=1, bias=0, distribution="normal"):
        if m is None:     # the reference calls xavier_init(self.output_proj) with output_proj=None
            return
        (nn.init.xavier_uniform_ if distribution == "uniform" else nn.init.xavier_normal_)(m.weight, gain=gain)
        if m.bias is not None:
            nn.init.constant_(m.bias, bias)

    def build_attention(cfg):
        return attention.build(cfg)

    def mod(name, **attrs):
        m = _Permissive(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    mod("mmcv", __path__=[])
    mod("mmcv.cnn", __path__=[], Linear=nn.Linear, xavier_init=xavier_init, constant_init=constant_init,
        bias_init_with_prob=lambda p: float(-torch.log(torch.tensor((1 - p) / p))))
    mod("mmcv.cnn.bricks", __path__=[])
    mod("mmcv.cnn.bricks.registry", ATTENTION=attention, TRANSFORMER_LAYER=layer,
        TRANSFORMER_LAYER_SEQUENCE=seq)
    mod("mmcv.cnn.bricks.transformer", build_attention=build_attention,
        TransformerLayerSequence=BaseModule)
    mod("mmcv.runner", __path__=[], force_fp32=_passthrough_decorator, auto_fp16=_passthrough_decorator,
        BaseModule=BaseModule)
    mod("mmcv.runner.base_module", BaseModule=BaseModule, ModuleList=nn.ModuleList, Sequential=nn.Sequential)
    mod("mmcv.utils", __path__=[], ext_loader=types.SimpleNamespace(load_ext=lambda *a, **k: _Anything()),
        TORCH_VERSION=torch.__version__, digit_version=lambda v: (1, 10, 0),
        deprecated_api_warning=lambda *a, **k: _passthrough_decorator)
    mod("mmcv.ops", __path__=[])
    mod("mmcv.ops.multi_scale_deform_attn", multi_scale_deformable_attn_pytorch=_msda_pytorch)
    for name in ("mmdet", "mmdet.models", "mmdet.models.utils", "mmdet3d", "mmdet3d.models",
                 "mmdet3d.models.losses"):
        mod(name, __path__=[])
    # decoder.py imports plotting libraries it never uses on this path
    for name in ("cv2", "matplotlib", "matplotlib.pyplot"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except ImportError:
                mod(name, __path__=[])

    pkg = types.ModuleType("vidar_ref")
    pkg.__path__ = [REF_BEVFORMER]
    sys.modules["vidar_ref"] = pkg
    for sub in ("modules", "dense_heads"):
        m = types.ModuleType(f"vidar_ref.{sub}")
        m.__path__ = [os.path.join(REF_BEVFORMER, sub)]
        sys.modules[f"vidar_ref.{sub}"] = m
    rays = types.ModuleType("vidar_ref.modules.ray_operations")
    rays.__path__ = [os.path.join(REF_BEVFORMER, "modules", "ray_operations")]
    sys.modules["vidar_ref.modules.ray_operations"] = rays
    # `from ..utils import e2e_predictor_utils` JIT-compiles CUDA at import: stub it out
    utils = _Permissive("vidar_ref.utils")
    utils.__path__ = []
    sys.modules["vidar_ref.utils"] = utils
    sys.modules["vidar_ref.utils.e2e_predictor_utils"] = _Permissive("vidar_ref.utils.e2e_predictor_utils")
    pkg.registries = dict(ATTENTION=attention)
    rays.LatentRendering = importlib.import_module(
        "vidar_ref.modules.ray_operations.latent_rendering").LatentRendering
    return pkg


def load_functions(relpath, names):
    """Execute ONLY the named top-level functions of a reference file (plus its plain imports that
    resolve here) and return them as a dict -- for files whose module body cannot run in this
    container (e2e_predictor_utils.py JIT-compiles CUDA extensions at import).  The source is read
    from /root/reference at call time; nothing is copied into the repo."""
    import ast
    path = os.path.join(REF_BEVFORMER, relpath)
    with open(path) as fh:
        tree = ast.parse(fh.read(), filename=path)
    ns = {"__name__": "vidar_ref._functions"}
    for node in tree.body:
        if isinstance(node, (ast.Import, ast.ImportFrom)) and not getattr(node, "level", 0):
            try:
                exec(compile(ast.Module([node], []), path, "exec"), ns)
            except ImportError:
                pass
        elif isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module([node], []), path, "exec"), ns)
    return {n: ns[n] for n in names}


def install_e2e_utils():
    """Put the pure helpers of utils/e2e_predictor_utils.py on the stub module the heads import."""
    install()
    stub = sys.modules["vidar_ref.utils.e2e_predictor_utils"]
    fns = load_functions(os.path.join("utils", "e2e_predictor_utils.py"),
                         ("coords_to_voxel_grids", "get_bev_grids", "get_bev_grids_3d", "get_inside_mask"))
    for k, v in fns.items():
        setattr(stub, k, v)
    sys.modules["vidar_ref.utils"].e2e_predictor_utils = stub      # `from ..utils import e2e_predictor_utils`
    return stub


def load(dotted):
    """e.g. load('modules.spatial_cross_attention') -> module object of the reference file."""
    install()
    return importlib.import_module(f"vidar_ref.{dotted}")


REF_PIPELINES = "/root/reference/projects/mmdet3d_plugin/datasets/pipelines"


def install_pipelines():
    """Load the reference's image transforms (datasets/pipelines/transform_3d.py and augmentation.py) with
    stand-ins for what they take from mmcv and mmdet: `bgr2hsv`, `hsv2bgr`, `imnormalize`, `impad`,
    `impad_to_multiple`, `parallel.DataContainer` and `datasets.builder.PIPELINES`.  The stand-ins restate mmcv 1.x's
    published definitions (mmcv/image/colorspace.py, photometric.py, geometric.py): the same cv2 calls with the same
    arguments.  -> {class name: class} of both files."""
    import numbers

    import cv2
    import numpy as np
    install()

    def imnormalize(img, mean, std, to_rgb=True):
        img = img.copy().astype(np.float32)
        assert img.dtype != np.uint8
        mean = np.float64(mean.reshape(1, -1))
        stdinv = 1 / np.float64(std.reshape(1, -1))
        if to_rgb:
            cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
        cv2.subtract(img, mean, img)
        cv2.multiply(img, stdinv, img)
        return img

    def impad(img, *, shape=None, padding=None, pad_val=0, padding_mode="constant"):
        assert (shape is not None) ^ (padding is not None)
        if shape is not None:
            padding = (0, 0, shape[1] - img.shape[1], shape[0] - img.shape[0])
        if isinstance(pad_val, tuple):
            assert len(pad_val) == img.shape[-1]
        elif not isinstance(pad_val, numbers.Number):
            raise TypeError(f"pad_val must be a int or a tuple. But received {type(pad_val)}")
        border = {"constant": cv2.BORDER_CONSTANT}[padding_mode]
        return cv2.copyMakeBorder(img, padding[1], padding[3], padding[0], padding[2], border, value=pad_val)

    def impad_to_multiple(img, divisor, pad_val=0):
        pad_h = int(np.ceil(img.shape[0] / divisor)) * divisor
        pad_w = int(np.ceil(img.shape[1] / divisor)) * divisor
        return impad(img, shape=(pad_h, pad_w), pad_val=pad_val)

    class DataContainer:
        def __init__(self, data, stack=False, padding_value=0, cpu_only=False, pad_dims=2):
            self.data, self.stack, self.cpu_only = data, stack, cpu_only

    mmcv = sys.modules["mmcv"]
    mmcv.bgr2hsv = lambda img: cv2.cvtColor(img, cv2.COLOR_BGR2HSV)
    mmcv.hsv2bgr = lambda img: cv2.cvtColor(img, cv2.COLOR_HSV2BGR)
    mmcv.imnormalize, mmcv.impad, mmcv.impad_to_multiple = imnormalize, impad, impad_to_multiple
    parallel = types.ModuleType("mmcv.parallel")
    parallel.DataContainer = DataContainer
    sys.modules["mmcv.parallel"] = parallel
    pipelines = _Registry()
    for name in ("mmdet.datasets", "mmdet.datasets.builder"):
        m = _Permissive(name)
        m.__path__ = []
        m.PIPELINES = pipelines
        sys.modules[name] = m
    for fname in ("transform_3d.py", "augmentation.py"):
        spec = importlib.util.spec_from_file_location(f"vidar_ref_pipelines_{fname[:-3]}",
                                                      os.path.join(REF_PIPELINES, fname))
        spec.loader.exec_module(importlib.util.module_from_spec(spec))
    return pipelines.modules
