"""The point half of ViDAR's pre-training samples on the H100 (vidar_1_8_nusc_3future.py:279-305, union2one of
nuscenes_vidar_dataset_v1.py:22-70, 199-200):

    LoadPointsFromFile -> CustomLoadPointsFromMultiSweeps -> CustomVoxelBasedPointSampler  (per queue frame)
      -> union2one: ego mask, last column := queue index, concatenation -> gt_points [sum M, 5]

The three classes take the reference's constructor arguments (mmdet3d 0.17.1's LoadPointsFromFile,
datasets/pipelines/loading.py:10-241).  Used as dataloader transforms, their `__call__(results)` does only the host
work: the file reads, the sweep selection, numpy's draws in the reference's order (`np.random.choice` when
`random_select`, then mmdet3d's two `np.random.shuffle` calls, made on int32 index vectors instead of the [N, 5]
point array: the same draws, the same generator state afterwards, a hundred times less work), and the survivor
counts of the remove-close / ego filter.  What to do to the points is recorded in `results['pts_aug']`.

`gather_gt_points(queue_results, ego_mask, device)` then builds a sample's `gt_points` from the recorded frames in
one device pass (csrc/point_pipeline.cu, include/vidar_b200.h §xi): the sweep transform, the filter, the merge, the
voxel sampler's first-occurrence selection, union2one's ego mask and queue-index column, bit for bit the reference.
Everything it needs goes up in one pinned, non-blocking copy.  No host sync, except with `compact=True`.
"""
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib

SEG_I, SEG_D, FRAME_I, FRAME_F, FRAME_G = 5, 17, 10, 6, 3
MAX_CELLS_PER_FRAME = 1 << 24


def read_points(path):
    """The float32 contents of a point file (mmcv's disk backend + np.frombuffer in mmdet3d)."""
    return np.fromfile(path, dtype=np.float32)


NUPLAN_FIELDS = ("x", "y", "z", "intensity", "ring", "lidar_info")
_PCD_TYPES = {"I": "int", "U": "uint", "F": "float"}


def parse_pcd(content, name="<bytes>"):
    """nuPlan's binary .pcd bytes -> float32 [N, 6] (x, y, z, intensity, ring, lidar_info): what
    `PointCloud.parse(...).to_pcd_bin2().T` gives (datasets/pipelines/nuplan_loading.py).  The header is read as
    PointCloud.parse_header reads it -- '#' lines skipped, one `KEY value...` per line up to DATA, a key with one
    value keeps it as a string -- and the same errors are raised: RuntimeError for a count other than 1, field lists
    of different lengths, data other than 'binary' or fewer point bytes than the header promises; KeyError for a
    missing header key; IndexError for a blank line or a header that ends before DATA.  Bytes after the points are
    ignored, as the reference ignores them."""
    pos, header = 0, {}
    while True:
        end = content.find(b"\n", pos)
        line = content[pos:] if end < 0 else content[pos:end + 1]
        pos = len(content) if end < 0 else end + 1
        line = line.decode("utf8").strip()
        if line.startswith("#"):
            continue
        cols = line.split()
        if not cols:
            raise IndexError(f"{name}: .pcd header: blank line or end of file before DATA")
        key = cols[0].lower()
        header[key] = cols[1:] if len(cols) > 2 else cols[1]
        if key == "data":
            break
    size = [int(v) for v in header["size"]]
    count = [int(v) for v in header["count"]]
    points = int(header["points"])
    for k in ("width", "height"):
        int(header[k])
    [int(v) for v in header["viewpoint"]]
    fields, types = list(header["fields"]), list(header["type"])
    header["version"]                                 # noqa: B018  (the header tuple needs every key)
    if any(c != 1 for c in count):
        raise RuntimeError(f'{name}: .pcd "count" has to be 1')
    if not len(fields) == len(size) == len(types) == len(count):
        raise RuntimeError(f"{name}: .pcd fields/size/type/count field number are inconsistent")
    if header["data"] != "binary":
        raise RuntimeError(f'{name}: .pcd data format {header["data"]!r} is not supported; "binary" is expected')
    row = np.dtype([(f, getattr(np, _PCD_TYPES[t] + str(int(sz) * 8))) for f, t, sz in zip(fields, types, size)])
    length = row.itemsize * points
    buf = content[pos:pos + length]
    if len(buf) != length:
        raise RuntimeError(f"{name}: incomplete .pcd stream: {length} bytes expected, {len(buf)} got")
    rec = np.frombuffer(buf, row)
    missing = [f for f in NUPLAN_FIELDS if f not in rec.dtype.names]
    if missing:
        raise ValueError(f"{name}: .pcd has no field {missing[0]!r} (nuPlan's six fields are {NUPLAN_FIELDS})")
    out = np.empty((points, len(NUPLAN_FIELDS)), np.float32)
    for j, f in enumerate(NUPLAN_FIELDS):
        out[:, j] = np.asarray(rec[f], dtype=np.float32)
    return out


def read_pcd(path):
    """parse_pcd of a .pcd file."""
    with open(path, "rb") as fh:
        return parse_pcd(fh.read(), path)


@dataclass
class Segment:
    """One source of a frame's merged cloud: the raw [n, 5] float32 array, the filter (None, or the ego box
    (x_lo, y_lo, x_hi, y_hi) as float32 with () for remove-close only), the sweep transform (float64 R, t, or None),
    the float32 time value and the number of points the filter keeps."""
    raw: np.ndarray
    filt: tuple = None
    R: np.ndarray = None
    t: np.ndarray = None
    time: np.float32 = np.float32(0)
    n_keep: int = 0
    time_col: bool = False             # 6 columns: column 4 is `time` (else the raw column 4)


@dataclass
class PointPlan:
    """What `gather_gt_points` does with one frame, recorded by the transforms in `results['pts_aug']`."""
    segments: list = field(default_factory=list)
    perm: np.ndarray = None            # int32 shuffled order of the current points, or None (no sampler)
    lo: np.ndarray = None              # float32 voxel range start (3)
    voxel_size: np.ndarray = None      # float32 (3)
    grid: tuple = None                 # voxel grid (x, y, z)
    max_voxels: int = 0

    def current(self):
        return [s for s in self.segments if s.time == 0]


def _check_dims(who, load_dim, use_dim):
    ud = list(range(use_dim)) if isinstance(use_dim, int) else list(use_dim)
    if load_dim != 5 or ud != [0, 1, 2, 3, 4]:
        raise ValueError(f"{who}: only load_dim=5 with use_dim=5 or [0, 1, 2, 3, 4] is supported (got {load_dim}, "
                         f"{use_dim})")


def _check_backend(who, file_client_args):
    if (file_client_args or {}).get("backend", "disk") != "disk":
        raise ValueError(f"{who}: only the 'disk' file backend is supported (got {file_client_args})")


class LoadPointsFromFile:
    """mmdet3d 0.17.1 LoadPointsFromFile: reads results['pts_filename'] into a float32 [N, load_dim] host array,
    results['points'].  The key frame stays on the host until `gather_gt_points`."""

    def __init__(self, coord_type, load_dim=6, use_dim=[0, 1, 2], shift_height=False, use_color=False,
                 file_client_args=dict(backend="disk")):
        if coord_type != "LIDAR" or shift_height or use_color:
            raise ValueError("LoadPointsFromFile: only coord_type='LIDAR' without shift_height / use_color is supported")
        _check_dims("LoadPointsFromFile", load_dim, use_dim)
        _check_backend("LoadPointsFromFile", file_client_args)
        self.coord_type, self.load_dim, self.use_dim = coord_type, load_dim, use_dim
        self.file_client_args = file_client_args

    def __call__(self, results):
        pts = read_points(results["pts_filename"]).reshape(-1, self.load_dim)
        results["points"] = pts
        results.pop("pts_aug", None)
        return results


class CustomLoadPointsFromMultiSweeps:
    """loading.py:10-223: selects the sweeps as the reference does (`np.random.choice` only when `random_select`
    and there are more sweeps than `sweeps_num`), loads them and counts the survivors of `_remove_close` with the
    reference's float32 comparisons.  Records one Segment per source in results['pts_aug']: the key frame (time 0),
    then the sweeps in `choices` order, or `sweeps_num` filtered copies of the key frame with `pad_empty_sweeps` and
    no sweeps.  With `hard_sweeps_timestamp` every segment's time is that value."""

    def __init__(self, ego_mask=None, hard_sweeps_timestamp=None, sweeps_num=10, load_dim=5, use_dim=[0, 1, 2, 4],
                 file_client_args=dict(backend="disk"), pad_empty_sweeps=False, remove_close=False,
                 random_select=True, load_future=False, test_mode=False):
        _check_dims("CustomLoadPointsFromMultiSweeps", load_dim, use_dim)
        _check_backend("CustomLoadPointsFromMultiSweeps", file_client_args)
        if ego_mask is not None and len(ego_mask) != 4:
            raise ValueError(f"CustomLoadPointsFromMultiSweeps: ego_mask needs 4 values (got {ego_mask})")
        self.ego_mask = ego_mask
        self.hard_sweeps_timestamp = hard_sweeps_timestamp
        self.load_dim, self.sweeps_num, self.use_dim = load_dim, sweeps_num, use_dim
        self.file_client_args = file_client_args
        self.pad_empty_sweeps, self.remove_close = pad_empty_sweeps, remove_close
        self.test_mode, self.random_select, self.load_future = test_mode, random_select, load_future

    def _select_index(self, sweeps, ts):
        if len(sweeps) <= self.sweeps_num:
            choices = np.arange(len(sweeps))
        elif self.test_mode:
            choices = np.arange(self.sweeps_num)
        elif self.random_select:
            choices = np.random.choice(len(sweeps), self.sweeps_num, replace=False)
        else:
            sweep_ts = np.array([sweep["timestamp"] for sweep in sweeps]) / 1e6
            choices = np.argsort(np.abs(sweep_ts - ts))[:self.sweeps_num]
        return choices

    def _filter(self):
        if not self.remove_close:
            return None
        return () if self.ego_mask is None else tuple(np.float32(v) for v in self.ego_mask)

    def __call__(self, results):
        key = results["points"]
        filt = self._filter()
        segs = [Segment(key, n_keep=key.shape[0])]
        ts = results["timestamp"]
        if self.pad_empty_sweeps and len(results["sweeps"]) == 0:
            for _ in range(self.sweeps_num):
                segs.append(Segment(key, filt))
        else:
            choices = self._select_index(results["sweeps"], ts)
            sweeps = results["sweeps"]
            if self.load_future:
                future_choices = self._select_index(results["future_sweeps"], ts) + len(sweeps)
                sweeps = list(sweeps) + list(results["future_sweeps"])
                choices = np.concatenate([choices, future_choices])
            for idx in choices:
                sweep = sweeps[idx]
                raw = read_points(sweep["data_path"]).reshape(-1, self.load_dim)
                segs.append(Segment(raw, filt, np.asarray(sweep["sensor2lidar_rotation"], np.float64),
                                    np.asarray(sweep["sensor2lidar_translation"], np.float64).reshape(3),
                                    np.float32(ts - sweep["timestamp"] / 1e6)))
        for s in segs[1:]:
            s.n_keep = count_kept(s.raw, s.filt)
        if self.hard_sweeps_timestamp is not None:
            for s in segs:
                s.time = np.float32(self.hard_sweeps_timestamp)
        results["pts_aug"] = PointPlan(segs)
        return results


class LoadNuPlanPointsFromFile:
    """nuplan_loading.py LoadNuPlanPointsFromFile: reads the nuPlan .pcd at results['pts_filename'] into a float32
    [N, 6] host array (x, y, z, intensity, ring, lidar_info), results['points'].  The parse runs here, in the
    loader's workers; the key frame stays on the host until `gather_gt_points`."""

    def __init__(self, coord_type):
        if coord_type not in ["LIDAR"]:
            raise ValueError(f"LoadNuPlanPointsFromFile: coord_type must be 'LIDAR' (got {coord_type!r})")
        self.coord_type = coord_type

    def __call__(self, results):
        results["points"] = read_pcd(results["pts_filename"])
        results.pop("pts_aug", None)
        return results


class LoadNuPlanPointsFromMultiSweeps(CustomLoadPointsFromMultiSweeps):
    """nuplan_loading.py LoadNuPlanPointsFromMultiSweeps over the plugin's LoadPointsFromMultiSweeps
    (loading.py:10-165) on the 6-column nuPlan points, with the same constructor arguments.  What the reference does:
      * the key frame's column 4 (ring) := 0, and each loaded sweep's column 4 := ts - sweep_ts: the time the voxel
        sampler's time_dim=4 reads.  Recorded as each segment's time, written to column 4 by `gather_gt_points`;
      * `_remove_close` (|x| < 1 and |y| < 1, then the ego box) only on sweeps and on the padded copies of the key
        frame -- never on the key frame itself.  With the configs' sweeps_num=0 no sweep is selected (nuPlan's
        results carry sweeps=[], and with pad_empty_sweeps the pad loop runs zero times), so neither filter removes
        a point here; union2one's ego mask in `gather_gt_points` is the one that does;
      * `hard_sweeps_timestamp` writes the LAST column (lidar_info), which union2one then overwrites with the queue
        index: it changes no output and is only checked.
    Sweep files are .pcd files read with parse_pcd and reshaped to `load_dim` columns, as the reference reshapes
    them, so loading a sweep needs load_dim=6."""

    def __init__(self, ego_mask=None, hard_sweeps_timestamp=None, sweeps_num=10, load_dim=5, use_dim=[0, 1, 2, 4],
                 file_client_args=dict(backend="disk"), pad_empty_sweeps=False, remove_close=False,
                 random_select=True, load_future=False, test_mode=False):
        ud = list(range(use_dim)) if isinstance(use_dim, int) else list(use_dim)
        if ud != [0, 1, 2, 3, 4, 5]:
            raise ValueError(f"LoadNuPlanPointsFromMultiSweeps: only use_dim=[0, 1, 2, 3, 4, 5] is supported (got "
                             f"{use_dim})")
        if sweeps_num > 0 and load_dim != 6:
            raise ValueError(f"LoadNuPlanPointsFromMultiSweeps: loading sweeps of nuPlan's 6 fields needs load_dim=6 "
                             f"(got {load_dim})")
        _check_backend("LoadNuPlanPointsFromMultiSweeps", file_client_args)
        if ego_mask is not None and len(ego_mask) != 4:
            raise ValueError(f"LoadNuPlanPointsFromMultiSweeps: ego_mask needs 4 values (got {ego_mask})")
        self.ego_mask = ego_mask
        self.hard_sweeps_timestamp = hard_sweeps_timestamp
        self.load_dim, self.sweeps_num, self.use_dim = load_dim, sweeps_num, use_dim
        self.file_client_args = file_client_args
        self.pad_empty_sweeps, self.remove_close = pad_empty_sweeps, remove_close
        self.test_mode, self.random_select, self.load_future = test_mode, random_select, load_future

    def __call__(self, results):
        key = results["points"]
        if not isinstance(key, np.ndarray) or key.dtype != np.float32 or key.ndim != 2 or key.shape[1] != 6:
            raise ValueError("LoadNuPlanPointsFromMultiSweeps: results['points'] must be LoadNuPlanPointsFromFile's "
                             "float32 [N, 6]")
        filt = self._filter()
        segs = [Segment(key, n_keep=key.shape[0], time_col=True)]
        ts = results["timestamp"]
        if self.pad_empty_sweeps and len(results["sweeps"]) == 0:
            for _ in range(self.sweeps_num):
                segs.append(Segment(key, filt, time_col=True))
        else:
            choices = self._select_index(results["sweeps"], ts)
            sweeps = results["sweeps"]
            if self.load_future:
                future_choices = self._select_index(results["future_sweeps"], ts) + len(sweeps)
                sweeps = list(sweeps) + list(results["future_sweeps"])
                choices = np.concatenate([choices, future_choices])
            for idx in choices:
                sweep = sweeps[idx]
                raw = read_pcd(sweep["data_path"]).reshape(-1, self.load_dim)
                segs.append(Segment(raw, filt, np.asarray(sweep["sensor2lidar_rotation"], np.float64),
                                    np.asarray(sweep["sensor2lidar_translation"], np.float64).reshape(3),
                                    np.float32(ts - sweep["timestamp"] / 1e6), time_col=True))
        for s in segs[1:]:
            s.n_keep = count_kept(s.raw, s.filt)
        results["pts_aug"] = PointPlan(segs)
        return results


def count_kept(raw, filt):
    """Points of raw [n, 5] that the reference's `_remove_close` keeps (all of them when filt is None)."""
    if filt is None:
        return raw.shape[0]
    x, y = raw[:, 0], raw[:, 1]
    keep = ~((np.abs(x) < 1.0) & (np.abs(y) < 1.0))
    if len(filt):
        keep &= ~((filt[0] <= x) & (filt[2] >= x) & (filt[1] <= y) & (filt[3] >= y))
    return int(np.count_nonzero(keep))


class CustomVoxelBasedPointSampler:
    """loading.py:226-241 over mmdet3d 0.17.1's VoxelBasedPointSampler.__call__: splits the merged points into the
    current (time == 0) and previous ones by segment, and makes mmdet3d's two `np.random.shuffle` draws on int32
    index vectors: the current points first, then the previous ones -- the current vector twice when there are no
    previous points, because mmdet3d then shuffles one array object through both names.  The previous points' draws
    are made and their points dropped, as mmdet3d drops them without a `prev_sweep_cfg`.  Records the current
    points' composed order and the VoxelGenerator parameters."""

    def __init__(self, cur_sweep_cfg, prev_sweep_cfg=None, time_dim=3):
        if prev_sweep_cfg is not None:
            raise ValueError("CustomVoxelBasedPointSampler: prev_sweep_cfg is not supported")
        if cur_sweep_cfg.get("max_num_points") != 1:
            raise ValueError(f"CustomVoxelBasedPointSampler: only max_num_points=1 is supported (got "
                             f"{cur_sweep_cfg.get('max_num_points')})")
        if time_dim != 4:
            raise ValueError(f"CustomVoxelBasedPointSampler: time_dim must be the time column, 4 (got {time_dim})")
        # mmdet3d's VoxelGenerator: float32 range and size, grid = round(f32(hi - lo) / vs)
        pcr = np.array(cur_sweep_cfg["point_cloud_range"], dtype=np.float32)
        vs = np.array(cur_sweep_cfg["voxel_size"], dtype=np.float32)
        grid = np.round((pcr[3:] - pcr[:3]) / vs).astype(np.int64)
        if grid.shape != (3,) or (grid <= 0).any() or int(np.prod(grid)) > MAX_CELLS_PER_FRAME:
            raise ValueError(f"CustomVoxelBasedPointSampler: voxel grid {grid.tolist()} must have 3 positive sides "
                             f"and at most {MAX_CELLS_PER_FRAME} cells")
        self.cur_sweep_cfg, self.prev_sweep_cfg, self.time_dim = cur_sweep_cfg, prev_sweep_cfg, time_dim
        self.lo, self.voxel_size, self.grid = pcr[:3].copy(), vs, tuple(int(g) for g in grid)
        self.max_voxels = int(cur_sweep_cfg.get("max_voxels", 20000))

    def __call__(self, results):
        plan = results.get("pts_aug")
        if not isinstance(plan, PointPlan):
            raise ValueError("CustomVoxelBasedPointSampler: results has no recorded multi-sweep points (run "
                             "CustomLoadPointsFromMultiSweeps first)")
        n_cur = sum(s.n_keep for s in plan.segments if s.time == 0)
        n_prev = sum(s.n_keep for s in plan.segments if s.time != 0)
        cur = np.arange(n_cur, dtype=np.int32)
        np.random.shuffle(cur)
        if n_prev == 0:
            np.random.shuffle(cur)
        else:
            np.random.shuffle(np.arange(n_prev, dtype=np.int32))
        plan.perm = cur
        plan.lo, plan.voxel_size, plan.grid, plan.max_voxels = self.lo, self.voxel_size, self.grid, self.max_voxels
        return results


def config_train_pipeline(point_cloud_range=(-51.2, -51.2, -5.0, 51.2, 51.2, 3.0), voxel_size=(1.0, 1.0, 1.0)):
    """The point transforms of the pre-training config's train_pipeline (vidar_1_8_nusc_3future.py:279-305).
    `voxel_size`: the voxel sampler's, 0.5 m in the 1-future configs (vidar_full_nusc_1future.py:291-295)."""
    return [LoadPointsFromFile(coord_type="LIDAR", load_dim=5, use_dim=5),
            CustomLoadPointsFromMultiSweeps(sweeps_num=2, use_dim=[0, 1, 2, 3, 4], pad_empty_sweeps=True,
                                            remove_close=True, ego_mask=(-0.8, -1.5, 0.8, 2.5),
                                            hard_sweeps_timestamp=0, random_select=False),
            CustomVoxelBasedPointSampler(cur_sweep_cfg=dict(max_num_points=1, point_cloud_range=list(point_cloud_range),
                                                            voxel_size=list(voxel_size), max_voxels=50000),
                                         time_dim=4)]


def config_test_pipeline():
    """The point transform of the config's test_pipeline (vidar_1_8_nusc_3future.py:319-324)."""
    return [LoadPointsFromFile(coord_type="LIDAR", load_dim=5, use_dim=5)]


def config_openscene_train_pipeline(point_cloud_range=(-51.2, -51.2, -5.0, 51.2, 51.2, 3.0)):
    """The point transforms of the OpenScene configs' train_pipeline (vidar_OpenScene_*_3future.py:274-296): the
    nuPlan loaders with sweeps_num=0, then the voxel sampler at 1 m."""
    return [LoadNuPlanPointsFromFile(coord_type="LIDAR"),
            LoadNuPlanPointsFromMultiSweeps(sweeps_num=0, use_dim=[0, 1, 2, 3, 4, 5], pad_empty_sweeps=True,
                                            remove_close=True, ego_mask=(-0.8, -1.5, 0.8, 2.5),
                                            hard_sweeps_timestamp=0, random_select=False),
            CustomVoxelBasedPointSampler(cur_sweep_cfg=dict(max_num_points=1, point_cloud_range=list(point_cloud_range),
                                                            voxel_size=[1.0, 1.0, 1.0], max_voxels=50000),
                                         time_dim=4)]


def config_openscene_test_pipeline():
    """The point transform of the OpenScene configs' test_pipeline (vidar_OpenScene_*_3future.py:307-308)."""
    return [LoadNuPlanPointsFromFile(coord_type="LIDAR")]


# ---------------------------------------------------------------------------------------------------------------
# device pass
# ---------------------------------------------------------------------------------------------------------------
def frame_plan(results):
    """The PointPlan of one frame's results; a frame that went through LoadPointsFromFile only (the test pipeline)
    is its key frame, kept whole and unsampled."""
    plan = results.get("pts_aug") if isinstance(results, dict) else None
    if isinstance(plan, PointPlan):
        return plan
    pts = results.get("points") if isinstance(results, dict) else None
    if not isinstance(pts, np.ndarray) or pts.dtype != np.float32 or pts.ndim != 2 or pts.shape[1] not in (5, 6):
        raise ValueError("gather_gt_points: every frame needs results['pts_aug'] from the transforms, or float32 "
                         "[N, 5] or [N, 6] results['points']")
    return PointPlan([Segment(pts, n_keep=pts.shape[0])])


class _Packer:
    """Lays the upload out in one byte buffer, each piece 16-byte aligned."""

    def __init__(self):
        self.parts, self.size = [], 0

    def add(self, a):
        a = np.ascontiguousarray(a)
        off = self.size
        self.parts.append((off, a))
        self.size = off + ((a.nbytes + 15) & ~15)
        return off


def pack(queue_results, ego_mask):
    """Host tables of one call -> (packer, {name: byte offset}, sizes dict).  Only the current segments go up: the
    previous sweeps' points are dropped by the sampler."""
    plans = [frame_plan(r) for r in queue_results]
    if not plans:
        raise ValueError("gather_gt_points: no frames")
    raws, raw_rows, cols = {}, 0, None
    seg_i, seg_d, frame_i, frame_f, frame_g, perms = [], [], [], [], [], []
    g = m = rows = cells = perm_off = 0
    for qi, plan in enumerate(plans):
        cur = plan.current() if plan.perm is not None else plan.segments
        g0, m0 = g, m
        for s in cur:
            if s.raw.dtype != np.float32 or s.raw.ndim != 2 or s.raw.shape[1] not in (5, 6):
                raise ValueError(f"gather_gt_points: raw points must be float32 [n, 5] or [n, 6] (got {s.raw.dtype} "
                                 f"{s.raw.shape})")
            if cols is not None and s.raw.shape[1] != cols:
                raise ValueError(f"gather_gt_points: raw points of {cols} and {s.raw.shape[1]} columns in one call")
            cols = s.raw.shape[1]
            if s.raw.shape[0] == 0:
                continue
            key = id(s.raw)
            if key not in raws:
                raws[key] = (raw_rows, s.raw)
                raw_rows += s.raw.shape[0]
            filt = 0 if s.filt is None else (2 if len(s.filt) else 1)
            seg_i.append((raws[key][0], s.raw.shape[0], g, filt, int(s.R is not None) | (2 if s.time_col else 0)))
            d = np.zeros(SEG_D)
            if s.R is not None:
                d[:9] = np.asarray(s.R, np.float64).reshape(9)
                d[9:12] = s.t
            if filt == 2:
                d[12:16] = s.filt
            d[16] = s.time
            seg_d.append(d)
            g += s.raw.shape[0]
            m += s.n_keep
        n_cur = m - m0
        voxel = plan.perm is not None
        if voxel and plan.perm.shape != (n_cur,):
            raise ValueError(f"gather_gt_points: frame {qi}'s order has {plan.perm.shape[0]} entries for {n_cur} "
                             "current points")
        cap = min(n_cur, plan.max_voxels) if voxel else n_cur
        fcells = int(np.prod(plan.grid)) if voxel else 0
        frame_i.append((m0, n_cur, rows, cap, qi, int(voxel), cells, perm_off, g0, g - g0))
        frame_f.append(np.concatenate([plan.lo, plan.voxel_size]) if voxel else np.zeros(6, np.float32))
        frame_g.append(plan.grid if voxel else (0, 0, 0))
        if voxel:
            perms.append(plan.perm.astype(np.int32, copy=False))
            perm_off += n_cur
        rows += cap
        cells += fcells
    if cols is None:                               # no points: the frames' own width
        cols = next((s.raw.shape[1] for p in plans for s in p.segments), 5)
    if not seg_i:                                  # a call with no points: one empty segment keeps the tables valid
        seg_i.append((0, 0, 0, 0, 0))
        seg_d.append(np.zeros(SEG_D))
    pk = _Packer()
    offs = dict(raw=pk.size)
    for off, raw in sorted(raws.values(), key=lambda v: v[0]):
        pk.parts.append((offs["raw"] + off * 4 * cols, np.ascontiguousarray(raw)))
    pk.size = offs["raw"] + ((raw_rows * 4 * cols + 15) & ~15)
    offs["seg_i"] = pk.add(np.asarray(seg_i, np.int64))
    offs["seg_d"] = pk.add(np.asarray(seg_d, np.float64))
    offs["frame_i"] = pk.add(np.asarray(frame_i, np.int64))
    offs["frame_f"] = pk.add(np.asarray(frame_f, np.float32))
    offs["frame_g"] = pk.add(np.asarray(frame_g, np.int64))
    offs["perm"] = pk.add(np.concatenate(perms) if perms else np.zeros(1, np.int32))
    ego = None if ego_mask is None else np.array([np.float32(v) for v in ego_mask], np.float32)
    if ego is not None and ego.shape != (4,):
        raise ValueError(f"gather_gt_points: ego_mask needs 4 values (got {ego_mask})")
    sizes = dict(S=len(seg_i), F=len(plans), n_g=g, n_cur=m, rows=rows, cells=cells, ego=ego, cols=cols,
                 raw_bytes=raw_rows * 4 * cols, perm_bytes=perm_off * 4)
    return pk, offs, sizes


def gather_gt_points(queue_results, ego_mask, device, compact=False, return_counts=False):
    """gt_points of one sample from its queue frames' results (in queue order; the queue index is the position in
    the list), on `device`'s current stream.

    Default: [1, R, C] float32 with R = the sum over frames of min(current points, max_voxels): each frame's rows in
    the reference's order, ego-masked and unused rows NaN.  C is the raw points' width: 5 for nuScenes (x, y, z,
    intensity, queue index), 6 for nuPlan (x, y, z, intensity, column 4, queue index: union2one overwrites the last
    column; column 4 is the multi-sweep step's time, or the raw ring without that step).  A NaN row belongs to no frame, so the heads' losses and
    evaluation take it as is; no host sync.  `compact=True`: exactly the reference's gt_points [sum M, C], after
    one sync for its size.  `return_counts=True` also returns int32 [F, 2] (device): each frame's merged points and
    sampled points as the device counted them."""
    pk, offs, sz = pack(queue_results, ego_mask)
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("gather_gt_points: device must be a CUDA device")
    host = torch.empty(pk.size, dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for off, a in pk.parts:
        hv[off:off + a.nbytes] = a.reshape(-1).view(np.uint8)
    with torch.cuda.device(device):
        buf = host.to(device, non_blocking=True)
        base = buf.data_ptr()
        rows = sz["rows"]
        cols = sz["cols"]
        out = torch.empty((rows, cols), dtype=torch.float32, device=device)
        counts = torch.empty((sz["F"], 2), dtype=torch.int32, device=device) if return_counts else None
        outc = torch.empty((rows, cols), dtype=torch.float32, device=device) if compact else None
        count = torch.empty(1, dtype=torch.int64, device=device) if compact else None

        def at(name):
            return base + offs[name]

        ego = sz["ego"]
        _lib.check(_lib.lib().vidar_point_pipeline_gather(
            at("raw"), at("seg_i"), at("seg_d"), sz["S"], at("frame_i"), at("frame_f"), at("frame_g"), sz["F"],
            at("perm"), sz["n_g"], sz["n_cur"], sz["cells"], None if ego is None else ego.ctypes.data,
            _lib.ptr(out) if rows else None, rows, _lib.ptr(counts), _lib.ptr(outc), _lib.ptr(count), cols,
            _lib.stream_ptr(device)))
    if compact:
        res = outc[: int(count.item())]
    else:
        res = out.view(1, rows, cols)
    return (res, counts) if return_counts else res


def upload_bytes(queue_results):
    """(bytes of raw points, bytes of int32 orders) that gather_gt_points uploads for these frames."""
    _, _, sz = pack(queue_results, None)
    return sz["raw_bytes"], sz["perm_bytes"]
