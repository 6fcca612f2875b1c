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


REF_DATASETS = "/root/reference/projects/mmdet3d_plugin/datasets"


def _load_methods(path, cls_name, names, ns):
    """Execute only the named methods of class `cls_name` in a reference file, as plain functions in `ns`."""
    import ast
    with open(path) as fh:
        tree = ast.parse(fh.read(), filename=path)
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == cls_name:
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in names:
                    exec(compile(ast.Module([item], []), path, "exec"), ns)
    return {n: ns[n] for n in names}


def install_point_pipelines(files=None):
    """Load the reference's point transforms (datasets/pipelines/loading.py) and NuScenesViDARDatasetV1's
    `_mask_points` / `union2one` (nuscenes_vidar_dataset_v1.py) with stand-ins for what they take from mmcv, mmdet,
    mmdet3d and nuscenes-devkit:
      * `mmcv.FileClient` (reads the file, or `files[path]` when a dict of preloaded bytes is given),
        `mmcv.check_file_exist`, `mmcv.parallel.DataContainer`, `mmdet.datasets.builder.PIPELINES`;
      * `BasePoints` / `LiDARPoints` (`tensor`, `shape`, `new_point`, `cat`, column and mask indexing) and
        `get_points_type`, restated from mmdet3d 0.17.1's core/points/base_points.py;
      * mmdet3d 0.17.1's `LoadPointsFromFile` and `VoxelBasedPointSampler`, with its `VoxelGenerator` /
        `points_to_voxel` / `_points_to_voxel_reverse_kernel` run by numba, restated from
        datasets/pipelines/loading.py, transforms_3d.py and core/voxel/voxel_generator.py;
      * `transform_matrix` and `Quaternion` (nuscenes-devkit / pyquaternion's definitions).
    mmdet3d is not part of the reference tree, so the voxel sampler step is checked against this restatement of
    upstream, not against upstream itself.
    -> dict of the classes and `union2one(previous_queue, future_queue, ego_mask)`."""
    import numba
    import numpy as np
    install()

    class FileClient:
        def __init__(self, backend="disk", **kw):
            self.backend = backend

        def get(self, path):
            if files is not None:
                return files[path]
            with open(path, "rb") as fh:
                return fh.read()

    class DataContainer:
        def __init__(self, data, stack=False, padding_value=0, cpu_only=False, pad_dims=2):
            self.data, self.stack, self.cpu_only = data, stack, cpu_only

    class BasePoints:
        def __init__(self, tensor, points_dim=3, attribute_dims=None):
            device = tensor.device if isinstance(tensor, torch.Tensor) else torch.device("cpu")
            tensor = torch.as_tensor(tensor, dtype=torch.float32, device=device)
            if tensor.numel() == 0:
                tensor = tensor.reshape((0, points_dim)).to(dtype=torch.float32, device=device)
            assert tensor.dim() == 2 and tensor.size(-1) == points_dim, tensor.size()
            self.tensor, self.points_dim, self.attribute_dims = tensor, points_dim, attribute_dims

        @property
        def shape(self):
            return self.tensor.shape

        @property
        def device(self):
            return self.tensor.device

        def new_point(self, data):
            new_tensor = self.tensor.new_tensor(data) if not isinstance(data, torch.Tensor) else data.to(self.device)
            return type(self)(new_tensor, points_dim=self.points_dim, attribute_dims=self.attribute_dims)

        @classmethod
        def cat(cls, points_list):
            return cls(torch.cat([p.tensor for p in points_list]), points_dim=points_list[0].tensor.shape[1],
                       attribute_dims=points_list[0].attribute_dims)

        def __len__(self):
            return self.tensor.shape[0]

        def __getitem__(self, item):
            if isinstance(item, tuple) and len(item) == 2:
                cols = item[1]
                if isinstance(cols, slice):
                    cols = list(range(cols.start or 0, self.tensor.shape[1] if cols.stop is None else cols.stop,
                                      cols.step or 1))
                elif isinstance(cols, int):
                    cols = [cols]
                p = self.tensor[item[0], cols]
            elif isinstance(item, (slice, np.ndarray, torch.Tensor)):
                p = self.tensor[item]
            else:
                raise NotImplementedError(type(item))
            return type(self)(p, points_dim=p.shape[1], attribute_dims=self.attribute_dims)

    class LiDARPoints(BasePoints):
        pass

    def get_points_type(points_type):
        assert points_type == "LIDAR", points_type
        return LiDARPoints

    @numba.jit(nopython=True)
    def _points_to_voxel_reverse_kernel(points, voxel_size, coors_range, num_points_per_voxel, coor_to_voxelidx,
                                        voxels, coors, max_points=35, max_voxels=20000):
        N = points.shape[0]
        ndim = 3
        ndim_minus_1 = ndim - 1
        grid_size = (coors_range[3:] - coors_range[:3]) / voxel_size
        grid_size = np.round(grid_size, 0, grid_size).astype(np.int32)
        coor = np.zeros(shape=(3, ), dtype=np.int32)
        voxel_num = 0
        failed = False
        for i in range(N):
            failed = False
            for j in range(ndim):
                c = np.floor((points[i, j] - coors_range[j]) / voxel_size[j])
                if c < 0 or c >= grid_size[j]:
                    failed = True
                    break
                coor[ndim_minus_1 - j] = c
            if failed:
                continue
            voxelidx = coor_to_voxelidx[coor[0], coor[1], coor[2]]
            if voxelidx == -1:
                voxelidx = voxel_num
                if voxel_num >= max_voxels:
                    continue
                voxel_num += 1
                coor_to_voxelidx[coor[0], coor[1], coor[2]] = voxelidx
                coors[voxelidx] = coor
            num = num_points_per_voxel[voxelidx]
            if num < max_points:
                voxels[voxelidx, num] = points[i]
                num_points_per_voxel[voxelidx] += 1
        return voxel_num

    def points_to_voxel(points, voxel_size, coors_range, max_points=35, reverse_index=True, max_voxels=20000):
        assert reverse_index
        voxelmap_shape = (coors_range[3:] - coors_range[:3]) / voxel_size
        voxelmap_shape = tuple(np.round(voxelmap_shape).astype(np.int32).tolist())[::-1]
        num_points_per_voxel = np.zeros(shape=(max_voxels, ), dtype=np.int32)
        coor_to_voxelidx = -np.ones(shape=voxelmap_shape, dtype=np.int32)
        voxels = np.zeros(shape=(max_voxels, max_points, points.shape[-1]), dtype=points.dtype)
        coors = np.zeros(shape=(max_voxels, 3), dtype=np.int32)
        voxel_num = _points_to_voxel_reverse_kernel(points, voxel_size, coors_range, num_points_per_voxel,
                                                    coor_to_voxelidx, voxels, coors, max_points, max_voxels)
        return voxels[:voxel_num], coors[:voxel_num], num_points_per_voxel[:voxel_num]

    class VoxelGenerator:
        def __init__(self, voxel_size, point_cloud_range, max_num_points, max_voxels=20000):
            point_cloud_range = np.array(point_cloud_range, dtype=np.float32)
            voxel_size = np.array(voxel_size, dtype=np.float32)
            grid_size = (point_cloud_range[3:] - point_cloud_range[:3]) / voxel_size
            self._voxel_size, self._point_cloud_range = voxel_size, point_cloud_range
            self._max_num_points, self._max_voxels = max_num_points, max_voxels
            self._grid_size = np.round(grid_size).astype(np.int64)

        def generate(self, points):
            return points_to_voxel(points, self._voxel_size, self._point_cloud_range, self._max_num_points, True,
                                   self._max_voxels)

    class VoxelBasedPointSampler:
        def __init__(self, cur_sweep_cfg, prev_sweep_cfg=None, time_dim=3):
            self.cur_voxel_generator = VoxelGenerator(**cur_sweep_cfg)
            self.cur_voxel_num = self.cur_voxel_generator._max_voxels
            self.time_dim = time_dim
            if prev_sweep_cfg is not None:
                assert prev_sweep_cfg["max_num_points"] == cur_sweep_cfg["max_num_points"]
                self.prev_voxel_generator = VoxelGenerator(**prev_sweep_cfg)
                self.prev_voxel_num = self.prev_voxel_generator._max_voxels
            else:
                self.prev_voxel_generator = None
                self.prev_voxel_num = 0

        def _sample_points(self, points, sampler, point_dim):
            voxels, coors, num_points_per_voxel = sampler.generate(points)
            if voxels.shape[0] < sampler._max_voxels:
                padding_points = np.zeros([sampler._max_voxels - voxels.shape[0], sampler._max_num_points,
                                           point_dim], dtype=points.dtype)
                padding_points[:] = voxels[0]
                sample_points = np.concatenate([voxels, padding_points], axis=0)
            else:
                sample_points = voxels
            return sample_points

        def __call__(self, results):
            points = results["points"]
            original_dim = points.shape[1]
            map_fields2dim = []
            start_dim = original_dim
            points_numpy = points.tensor.numpy()
            extra_channel = [points_numpy]
            for idx, key in enumerate(results["pts_mask_fields"]):
                map_fields2dim.append((key, idx + start_dim))
                extra_channel.append(results[key][..., None])
            start_dim += len(results["pts_mask_fields"])
            for idx, key in enumerate(results["pts_seg_fields"]):
                map_fields2dim.append((key, idx + start_dim))
                extra_channel.append(results[key][..., None])
            points_numpy = np.concatenate(extra_channel, axis=-1)
            cur_points_flag = (points_numpy[:, self.time_dim] == 0)
            cur_sweep_points = points_numpy[cur_points_flag]
            prev_sweeps_points = points_numpy[~cur_points_flag]
            if prev_sweeps_points.shape[0] == 0:
                prev_sweeps_points = cur_sweep_points
            np.random.shuffle(cur_sweep_points)
            np.random.shuffle(prev_sweeps_points)
            cur_sweep_points = self._sample_points(cur_sweep_points, self.cur_voxel_generator,
                                                   points_numpy.shape[1])
            if self.prev_voxel_generator is not None:
                prev_sweeps_points = self._sample_points(prev_sweeps_points, self.prev_voxel_generator,
                                                         points_numpy.shape[1])
                points_numpy = np.concatenate([cur_sweep_points, prev_sweeps_points], 0)
            else:
                points_numpy = cur_sweep_points
            if self.cur_voxel_generator._max_num_points == 1:
                points_numpy = points_numpy.squeeze(1)
            results["points"] = points.new_point(points_numpy[..., :original_dim])
            for key, dim_index in map_fields2dim:
                results[key] = points_numpy[..., dim_index]
            return results

    class LoadPointsFromFile:
        def __init__(self, coord_type, load_dim=6, use_dim=[0, 1, 2], shift_height=False, use_color=False,
                     file_client_args=dict(backend="disk")):
            assert not shift_height and not use_color
            if isinstance(use_dim, int):
                use_dim = list(range(use_dim))
            assert max(use_dim) < load_dim
            self.coord_type, self.load_dim, self.use_dim = coord_type, load_dim, use_dim
            self.file_client_args = file_client_args.copy()
            self.file_client = None

        def _load_points(self, pts_filename):
            if self.file_client is None:
                self.file_client = FileClient(**self.file_client_args)
            return np.frombuffer(self.file_client.get(pts_filename), dtype=np.float32)

        def __call__(self, results):
            points = self._load_points(results["pts_filename"])
            points = points.reshape(-1, self.load_dim)
            points = points[:, self.use_dim]
            points = get_points_type(self.coord_type)(points, points_dim=points.shape[-1], attribute_dims=None)
            results["points"] = points
            return results

    class Quaternion:
        def __init__(self, q):
            self.q = np.asarray(q, np.float64)

        @property
        def rotation_matrix(self):
            w, x, y, z = self.q / np.linalg.norm(self.q)
            return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                             [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                             [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])

    def transform_matrix(translation=np.array([0, 0, 0]), rotation=Quaternion([1, 0, 0, 0]), inverse=False):
        tm = np.eye(4)
        if inverse:
            rot_inv = rotation.rotation_matrix.T
            tm[:3, :3] = rot_inv
            tm[:3, 3] = rot_inv.dot(np.transpose(-np.array(translation)))
        else:
            tm[:3, :3] = rotation.rotation_matrix
            tm[:3, 3] = np.transpose(np.array(translation))
        return tm

    mmcv = sys.modules["mmcv"]
    mmcv.FileClient = FileClient
    mmcv.check_file_exist = lambda *a, **k: None
    parallel = types.ModuleType("mmcv.parallel")
    parallel.DataContainer = DataContainer
    sys.modules["mmcv.parallel"] = parallel
    pipelines = _Registry()
    for name in ("mmdet.datasets", "mmdet.datasets.builder"):
        m = _Permissive(name)
        m.__path__ = []
        m.PIPELINES = pipelines
        sys.modules[name] = m
    points_mod = types.ModuleType("mmdet3d.core.points")
    points_mod.BasePoints, points_mod.LiDARPoints, points_mod.get_points_type = BasePoints, LiDARPoints, get_points_type
    sys.modules["mmdet3d.core"] = _Permissive("mmdet3d.core")
    sys.modules["mmdet3d.core"].__path__ = []
    sys.modules["mmdet3d.core.points"] = points_mod
    dp = types.ModuleType("mmdet3d.datasets.pipelines")
    dp.VoxelBasedPointSampler = VoxelBasedPointSampler
    sys.modules["mmdet3d.datasets"] = _Permissive("mmdet3d.datasets")
    sys.modules["mmdet3d.datasets"].__path__ = []
    sys.modules["mmdet3d.datasets.pipelines"] = dp
    spec = importlib.util.spec_from_file_location("vidar_ref_pipelines_loading", os.path.join(REF_PIPELINES, "loading.py"))
    loading = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(loading)
    sys.modules["vidar_ref_pipelines_loading"] = loading

    ns = dict(np=np, torch=torch, copy=__import__("copy"), DC=DataContainer, transform_matrix=transform_matrix,
              Quaternion=Quaternion)
    meths = _load_methods(os.path.join(REF_DATASETS, "nuscenes_vidar_dataset_v1.py"), "NuScenesViDARDatasetV1",
                          ("_mask_points", "union2one"), ns)

    class _Dataset:
        _mask_points = meths["_mask_points"]
        union2one = meths["union2one"]

    def union2one(previous_queue, future_queue, ego_mask):
        ds = _Dataset()
        ds.ego_mask, ds.future_length = ego_mask, len(future_queue) - 1
        return ds.union2one(previous_queue, future_queue)

    return dict(LoadPointsFromFile=LoadPointsFromFile,
                CustomLoadPointsFromMultiSweeps=loading.CustomLoadPointsFromMultiSweeps,
                CustomVoxelBasedPointSampler=loading.CustomVoxelBasedPointSampler, LiDARPoints=LiDARPoints,
                DataContainer=DataContainer, union2one=union2one, transform_matrix=transform_matrix,
                Quaternion=Quaternion)


def install_nuplan_pipelines():
    """Load the reference's nuPlan point loaders (datasets/pipelines/nuplan_loading.py: `PointCloud`,
    `LoadNuPlanPointsFromFile`, `LoadNuPlanPointsFromMultiSweeps` over loading.py's LoadPointsFromMultiSweeps) and
    NuPlanViDARDatasetV1's `_mask_points` / `union2one`, on the stand-ins of `install_point_pipelines`.
    -> that dict with these names added."""
    import numpy as np
    ref = install_point_pipelines()
    pkg = types.ModuleType("vidar_ref_nuplan")
    pkg.__path__ = [REF_PIPELINES]
    sys.modules["vidar_ref_nuplan"] = pkg
    sys.modules["vidar_ref_nuplan.loading"] = sys.modules.get("vidar_ref_pipelines_loading") or _load_loading()
    spec = importlib.util.spec_from_file_location("vidar_ref_nuplan.nuplan_loading",
                                                  os.path.join(REF_PIPELINES, "nuplan_loading.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    ns = dict(np=np, torch=torch, copy=__import__("copy"), DC=ref["DataContainer"],
              transform_matrix=ref["transform_matrix"], Quaternion=ref["Quaternion"])
    meths = _load_methods(os.path.join(REF_DATASETS, "nuplan_vidar_dataset_v1.py"), "NuPlanViDARDatasetV1",
                          ("_mask_points", "union2one"), ns)

    class _Dataset:
        _mask_points = meths["_mask_points"]
        union2one = meths["union2one"]

    def union2one(previous_queue, future_queue, ego_mask):
        ds = _Dataset()
        ds.ego_mask, ds.future_length = ego_mask, len(future_queue) - 1
        return ds.union2one(previous_queue, future_queue)

    return dict(ref, PointCloud=mod.PointCloud, LoadNuPlanPointsFromFile=mod.LoadNuPlanPointsFromFile,
                LoadNuPlanPointsFromMultiSweeps=mod.LoadNuPlanPointsFromMultiSweeps, nuplan_union2one=union2one)


def _load_loading():
    spec = importlib.util.spec_from_file_location("vidar_ref_nuplan.loading", os.path.join(REF_PIPELINES, "loading.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def install_scale_pipeline():
    """The reference's RandomScaleImageMultiViewImage (transform_3d.py), with mmcv.imresize restated from mmcv 1.x
    (mmcv/image/geometric.py): cv2.resize(img, size, interpolation=cv2.INTER_LINEAR), the 'bilinear' default."""
    import cv2
    classes = install_pipelines()
    sys.modules["mmcv"].imresize = lambda img, size, return_scale=False, interpolation="bilinear": cv2.resize(
        img, size, interpolation={"bilinear": cv2.INTER_LINEAR}[interpolation])
    return classes["RandomScaleImageMultiViewImage"]
