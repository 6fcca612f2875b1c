"""Ego motion in the pre-training graph: each frame's pose metas, as the nuScenes ViDAR dataset makes them, and the
device ops that align the BEV of one frame to the next (`SyntheticViDAR(ego_motion=True)`).

Host, float64 numpy, as the reference computes them before its pipeline:
  * `frame_can_bus`: get_data_info's can_bus fill (datasets/nuscenes_dataset.py:156-163, 215-225): translation and
    rotation over can_bus[0:7], the patch angle (yaw in [0, 360)) in radians at [-2] and degrees at [-1], and
    lidar2global_rotation = ego2global R @ lidar2ego R;
  * `queue_metas`: union2one's metas (datasets/nuscenes_vidar_dataset_v1.py:38-205) of one queue: each image frame's
    can_bus as deltas to the previous frame (zeros and prev_bev_exists=False at a scene start), its
    ref_lidar_to_cur_lidar, and for the current frame future_can_bus, future2ref / ref2future_lidar_transform and
    total_cur2ref / total_ref2cur_lidar_transform.
pyquaternion and the nuScenes devkit are not dependencies: `Quaternion.rotation_matrix`, `transform_matrix` and
`quaternion_yaw` are restated from their published definitions (pyquaternion's q_matrix @ q_bar_matrix^T product,
nuscenes.utils.geometry_utils.transform_matrix, nuscenes.eval.common.utils.quaternion_yaw).  The goldens check the
metas against the reference's union2one run over these same helpers, so they pin the dataset's statements; that
the helpers equal the packages' bit for bit rests on the restatement alone (a weaker pin).

Device:
  * `bev_shift`: get_bev_features' shift of the history reference points (modules/transformer.py:121-135);
  * `rotation_rows`: the row map of torchvision's nearest `rotate(prev_bev [C, H, W], angle, center=[100, 100])`
    (transformer.py:137-150), built by running torchvision's own grid statements on a one-channel image of cell
    indices, so it selects exactly what the rotation selects on that device;
  * `rotate_stack`: TSA's value [bs * 2, Q, C] = [rotated previous BEV, query] in one kernel (csrc/bev_rotate.cu,
    include/vidar_b200.h §xv), with a deterministic backward;
  * `future_grids`: `_align_bev_coordnates` (detectors/vidar.py:196-238): each future frame's BEV grid moved into
    the previous frame's coordinates;
  * `future_inputs`: every future roll-out's can_bus and moved grid from the current frame's metas.
Every host-made value reaches the device through a pinned, non-blocking upload: no host sync.
"""
import copy

import numpy as np
import torch
from torch.autograd.function import Function, once_differentiable

from . import _lib

ROTATE_CENTER = (100, 100)       # PerceptionTransformer's rotate_center, the same at every BEV size
GRID_LENGTH = (0.512, 0.512)     # get_bev_features' grid_length default
POSE_KEYS = ("ego2global_translation", "ego2global_rotation", "lidar2ego_translation", "lidar2ego_rotation",
             "can_bus", "scene_token")
CAN_BUS_DIMS = (0, 1, 2, 17)     # the future head's can_bus_dims (vidar_1_8_nusc_3future.py:125)


# ------------------------------------------------------------------------------------------------
# restated pose helpers (pyquaternion, nuScenes devkit)
# ------------------------------------------------------------------------------------------------
class Quaternion:
    """pyquaternion.Quaternion(w, x, y, z) as far as the dataset uses it: construction from 4 numbers and
    `rotation_matrix` (normalised unless already unit to 1e-14, then q_matrix @ q_bar_matrix^T, lower 3 x 3)."""

    def __init__(self, q):
        self.q = np.array(q, dtype=float).reshape(4)

    def _q_matrix(self):
        q = self.q
        return np.array([[q[0], -q[1], -q[2], -q[3]],
                         [q[1], q[0], -q[3], q[2]],
                         [q[2], q[3], q[0], -q[1]],
                         [q[3], -q[2], q[1], q[0]]])

    def _q_bar_matrix(self):
        q = self.q
        return np.array([[q[0], -q[1], -q[2], -q[3]],
                         [q[1], q[0], q[3], -q[2]],
                         [q[2], -q[3], q[0], q[1]],
                         [q[3], q[2], -q[1], q[0]]])

    def _normalise(self):
        if not abs(1.0 - np.dot(self.q, self.q)) < 1e-14:
            n = np.sqrt(np.dot(self.q, self.q))
            if n > 0:
                self.q = self.q / n

    @property
    def rotation_matrix(self):
        self._normalise()
        return np.dot(self._q_matrix(), self._q_bar_matrix().conj().transpose())[1:][:, 1:]

    def __array__(self, dtype=None, copy=None):
        return self.q if dtype is None else self.q.astype(dtype)


def transform_matrix(translation=np.array([0, 0, 0]), rotation=Quaternion([1, 0, 0, 0]), inverse=False):
    """nuscenes.utils.geometry_utils.transform_matrix."""
    tm = np.eye(4)
    if inverse:
        rot_inv = rotation.rotation_matrix.T
        trans = np.transpose(-np.array(translation))
        tm[:3, :3] = rot_inv
        tm[:3, 3] = rot_inv.dot(trans)
    else:
        tm[:3, :3] = rotation.rotation_matrix
        tm[:3, 3] = np.transpose(np.array(translation))
    return tm


def quaternion_yaw(q):
    """nuscenes.eval.common.utils.quaternion_yaw: the yaw of q's x axis projected on the xy plane."""
    v = np.dot(q.rotation_matrix, np.array([1, 0, 0]))
    return np.arctan2(v[1], v[0])


# ------------------------------------------------------------------------------------------------
# metas of a queue (host)
# ------------------------------------------------------------------------------------------------
def _require_pose(frame, where):
    for key in POSE_KEYS:
        if key not in frame:
            raise ValueError(f"ego motion: {where} has no {key!r} (a pose needs {', '.join(POSE_KEYS)})")


def frame_can_bus(frame):
    """get_data_info's pose fields of one frame -> dict(can_bus float64 [18] with the ego pose and patch angle filled,
    lidar2global_rotation [3, 3], and the frame's pose keys)."""
    lidar2ego = np.eye(4)
    lidar2ego[:3, :3] = Quaternion(frame["lidar2ego_rotation"]).rotation_matrix
    lidar2ego[:3, 3] = np.array(frame["lidar2ego_translation"])
    ego2global = np.eye(4)
    ego2global[:3, :3] = Quaternion(frame["ego2global_rotation"]).rotation_matrix
    ego2global[:3, 3] = np.array(frame["ego2global_translation"])
    rotation = Quaternion(frame["ego2global_rotation"])
    can_bus = np.array(frame["can_bus"], dtype=np.float64).copy()
    if can_bus.shape != (18,):
        raise ValueError(f"ego motion: can_bus must hold 18 values (got shape {can_bus.shape})")
    can_bus[:3] = frame["ego2global_translation"]
    can_bus[3:7] = rotation
    patch_angle = quaternion_yaw(rotation) / np.pi * 180
    if patch_angle < 0:
        patch_angle += 360
    can_bus[-2] = patch_angle / 180 * np.pi
    can_bus[-1] = patch_angle
    return dict(can_bus=can_bus, lidar2global_rotation=ego2global[:3, :3] @ lidar2ego[:3, :3],
                scene_token=frame["scene_token"], ego2global_translation=frame["ego2global_translation"],
                ego2global_rotation=frame["ego2global_rotation"], lidar2ego_translation=frame["lidar2ego_translation"],
                lidar2ego_rotation=frame["lidar2ego_rotation"])


def queue_metas(queue):
    """A queue of results dicts (oldest first: the image frames -- history and current --, then the GT-only future
    frames; every frame with the `POSE_KEYS`) -> [metas] of the image frames: union2one's can_bus, prev_bev_exists,
    lidar2global_rotation and ref_lidar_to_cur_lidar, and on the current frame future_can_bus [1 + F, 18],
    future2ref / ref2future_lidar_transform [1 + F, 4, 4] and total_cur2ref / total_ref2cur_lidar_transform
    [T + F, 4, 4] (F future frames).  A future frame from another scene than the current one is an error."""
    for i, f in enumerate(queue):
        _require_pose(f, f"queue frame {i}")
    num_images = sum("img_filename" in f for f in queue)
    if num_images < 1 or any("img_filename" not in f for f in queue[:num_images]):
        raise ValueError("ego motion: a queue holds its image frames first, then the future frames")
    metas = [frame_can_bus(f) for f in queue]
    previous, future = metas[:num_images], metas[num_images - 1:]
    ref = previous[-1]
    ref_e2g = Quaternion(ref["ego2global_rotation"])
    ref_g2e_transform = transform_matrix(ref["ego2global_translation"], ref_e2g, inverse=True)
    ref_e2g_transform = transform_matrix(ref["ego2global_translation"], ref_e2g, inverse=False)
    ref_l2e = Quaternion(ref["lidar2ego_rotation"])
    ref_l2e_transform = transform_matrix(ref["lidar2ego_translation"], ref_l2e, inverse=False)
    ref_e2l_transform = transform_matrix(ref["lidar2ego_translation"], ref_l2e, inverse=True)
    cur2ref, ref2cur = [], []
    for meta in previous[:-1] + future:
        e2g = Quaternion(meta["ego2global_rotation"])
        l2e = Quaternion(meta["lidar2ego_rotation"])
        curr_e2g_transform = transform_matrix(meta["ego2global_translation"], e2g, inverse=False)
        curr_g2e_transform = transform_matrix(meta["ego2global_translation"], e2g, inverse=True)
        curr_l2e_transform = transform_matrix(meta["lidar2ego_translation"], l2e, inverse=False)
        curr_e2l_transform = transform_matrix(meta["lidar2ego_translation"], l2e, inverse=True)
        cur2ref.append(curr_l2e_transform.T @ curr_e2g_transform.T @ ref_g2e_transform.T @ ref_e2l_transform.T)
        ref2cur.append(ref_l2e_transform.T @ ref_e2g_transform.T @ curr_g2e_transform.T @ curr_e2l_transform.T)

    out = []
    prev_scene, prev_pos, prev_angle = None, None, None
    for i, meta in enumerate(previous):
        can_bus = meta["can_bus"].copy()
        pos, angle = copy.deepcopy(can_bus[:3]), copy.deepcopy(can_bus[-1])
        exists = meta["scene_token"] == prev_scene
        if exists:
            can_bus[:3] = pos - prev_pos
            can_bus[-1] = angle - prev_angle
        else:
            prev_scene = meta["scene_token"]
            can_bus[:3] = 0
            can_bus[-1] = 0
        prev_pos, prev_angle = pos, angle
        out.append(dict(can_bus=can_bus, prev_bev_exists=exists, lidar2global_rotation=meta["lidar2global_rotation"],
                        ref_lidar_to_cur_lidar=ref2cur[i], scene_token=meta["scene_token"]))

    future_can_bus, future2ref, ref2future, ref_can_bus = [], [], [], None
    for i, meta in enumerate(future):
        if meta["scene_token"] != ref["scene_token"]:
            raise ValueError(f"ego motion: future frame {i} is from another scene than the current frame")
        future2ref.append(cur2ref[i + num_images - 1])
        ref2future.append(ref2cur[i + num_images - 1])
        # future_queue[0] is the current frame's own results dict (_prepare_data_info builds it apart from the
        # history's), so its can_bus here is the absolute one, not the history loop's deltas
        can_bus = meta["can_bus"]
        new_can_bus = can_bus.copy()
        if i == 0:
            new_can_bus[:3] = 0
            new_can_bus[-1] = 0
        else:
            pos = np.array([0, 0, 0, 1]).reshape(1, 4) @ future2ref[-1] @ ref2future[-2]
            new_can_bus[:3] = pos[:, :3]
            new_can_bus[-1] = can_bus[-1] - ref_can_bus[-1]
        future_can_bus.append(new_can_bus)
        ref_can_bus = can_bus.copy()
    out[-1].update(future_can_bus=np.array(future_can_bus), future2ref_lidar_transform=np.array(future2ref),
                   ref2future_lidar_transform=np.array(ref2future),
                   total_cur2ref_lidar_transform=np.array(cur2ref), total_ref2cur_lidar_transform=np.array(ref2cur))
    return out


def require_metas(metas, future_frames=0):
    """Check one image frame's metas for the ego-motion graph; `future_frames` > 0: the current frame's future
    fields too.  Raises ValueError naming the first missing key."""
    keys = ["can_bus", "prev_bev_exists", "lidar2global_rotation", "ref_lidar_to_cur_lidar"]
    if future_frames:
        keys += ["future_can_bus", "future2ref_lidar_transform", "ref2future_lidar_transform"]
    for m in metas:
        for key in keys:
            if key not in m:
                raise ValueError(f"ego motion: img_metas has no {key!r} (build them with ego_motion.queue_metas)")
        if future_frames and len(m["future_can_bus"]) < 1 + future_frames:
            raise ValueError(f"ego motion: {future_frames} future frames need {1 + future_frames} future_can_bus rows "
                             f"(got {len(m['future_can_bus'])})")


# ------------------------------------------------------------------------------------------------
# encoder and decoder alignment
# ------------------------------------------------------------------------------------------------
def bev_shift(metas, bev_h, bev_w):
    """get_bev_features' shift (transformer.py:121-134): the can_bus translation in the lidar frame over the grid
    length and BEV size -> float64 [bs, 2] (x, y) on the host."""
    delta_global = np.array([m["can_bus"][:3] for m in metas])
    rot = np.array([m["lidar2global_rotation"] for m in metas])
    delta_lidar = np.array([np.linalg.inv(rot[i]) @ delta_global[i] for i in range(len(metas))])
    shift_y = delta_lidar[:, 1] / GRID_LENGTH[0] / bev_h
    shift_x = delta_lidar[:, 0] / GRID_LENGTH[1] / bev_w
    return np.stack([shift_x, shift_y], 1)


def upload(array, device, dtype=torch.float32):
    """A host array on `device` in `dtype` (cast on the host, as new_tensor casts), through pinned memory without
    blocking."""
    t = torch.from_numpy(np.ascontiguousarray(array)).to(dtype)
    return t.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else t.to(device)


def rotation_rows(angles, bev_h, bev_w, device):
    """The row map of torchvision's `rotate(img [C, bev_h, bev_w], angle, center=ROTATE_CENTER)` (nearest, zero
    fill) for each angle (degrees) -> int32 [len(angles), bev_h * bev_w]: output cell q takes source cell rows[q], or
    zero where rows[q] = -1.  torchvision's statements -- its inverse affine matrix on the host, then
    `_gen_affine_grid` and grid_sample on the device -- run here on an image of cell index + 1 (exact in fp32 up to
    2^24 cells), with the matrix uploaded pinned instead of by torch.tensor (a blocking copy)."""
    from torchvision.transforms.functional import _get_inverse_affine_matrix
    if bev_h * bev_w >= 1 << 24:
        raise ValueError(f"rotation_rows: {bev_h} x {bev_w} cells cannot be indexed exactly in fp32")
    center_f = [1.0 * (c - s * 0.5) for c, s in zip(ROTATE_CENTER, [bev_w, bev_h])]
    host = np.array([_get_inverse_affine_matrix(center_f, -float(a), [0.0, 0.0], 1.0, [0.0, 0.0]) + [0.5 * bev_w,
                                                                                                     0.5 * bev_h]
                     for a in angles], np.float64)
    buf = upload(host, device)                                              # [n, 8]: theta (2 x 3), 0.5 w, 0.5 h
    n = len(angles)
    theta = buf[:, :6].reshape(n, 2, 3)
    d = 0.5                                                                  # torchvision's _gen_affine_grid
    base_grid = torch.empty(1, bev_h, bev_w, 3, dtype=theta.dtype, device=device)
    x_grid = torch.linspace(-bev_w * 0.5 + d, bev_w * 0.5 + d - 1, steps=bev_w, device=device)
    base_grid[..., 0].copy_(x_grid)
    y_grid = torch.linspace(-bev_h * 0.5 + d, bev_h * 0.5 + d - 1, steps=bev_h, device=device).unsqueeze_(-1)
    base_grid[..., 1].copy_(y_grid)
    base_grid[..., 2].fill_(1)
    index = (torch.arange(bev_h * bev_w, device=device, dtype=torch.float32) + 1).view(1, 1, bev_h, bev_w)
    rows = []
    for i in range(n):
        rescaled_theta = theta[i:i + 1].transpose(1, 2) / buf[i, 6:8]
        grid = base_grid.view(1, bev_h * bev_w, 3).bmm(rescaled_theta).view(1, bev_h, bev_w, 2)
        img = torch.nn.functional.grid_sample(index, grid, mode="nearest", padding_mode="zeros", align_corners=False)
        rows.append(img.view(-1).to(torch.int32) - 1)
    return torch.stack(rows)


def _check_stack(prev, query, rows):
    if prev.dim() != 3 or query.shape != prev.shape:
        raise ValueError(f"rotate_stack: prev and query must be [bs, Q, C] alike (got {tuple(prev.shape)}, "
                         f"{tuple(query.shape)})")
    if rows.dtype != torch.int32 or tuple(rows.shape) != tuple(prev.shape[:2]):
        raise ValueError(f"rotate_stack: rows must be int32 [bs, Q] (got {rows.dtype} {tuple(rows.shape)})")
    if prev.dtype != torch.float32 or query.dtype != torch.float32 or prev.shape[2] % 4:
        raise ValueError(f"rotate_stack: fp32 features with C a multiple of 4 (got {prev.dtype}, {query.dtype}, "
                         f"C {prev.shape[2]})")


class RotateStack(Function):
    """apply(prev [bs, Q, C], query [bs, Q, C], rows [bs, Q] int32) -> value [bs * 2, Q, C] (csrc/bev_rotate.cu)."""

    @staticmethod
    def forward(ctx, prev, query, rows):
        _check_stack(prev, query, rows)
        prev, query, rows = _lib.aligned(prev.contiguous()), _lib.aligned(query.contiguous()), rows.contiguous()
        _lib.require_cuda(prev=prev, query=query, rows=rows)
        bs, Q, C = prev.shape
        value = torch.empty((bs * 2, Q, C), dtype=prev.dtype, device=prev.device)
        with torch.cuda.device(prev.device):
            _lib.check(_lib.lib().vidar_bev_rotate_stack_forward(
                _lib.ptr(prev), _lib.ptr(query), _lib.ptr(rows), _lib.ptr(value), bs, Q, C,
                _lib.stream_ptr(prev.device)))
        ctx.save_for_backward(rows)
        return value

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_value):
        rows, = ctx.saved_tensors
        g = _lib.aligned(grad_value.contiguous())
        bs, Q = rows.shape
        C = g.shape[2]
        grad_prev = torch.empty((bs, Q, C), dtype=g.dtype, device=g.device)
        grad_query = torch.empty_like(grad_prev)
        with torch.cuda.device(g.device):
            _lib.check(_lib.lib().vidar_bev_rotate_stack_backward(
                _lib.ptr(g), _lib.ptr(rows), _lib.ptr(grad_prev), _lib.ptr(grad_query), bs, Q, C,
                _lib.stream_ptr(g.device)))
        return grad_prev, grad_query, None


def rotate_stack(prev, query, rows):
    """TSA's value with the previous BEV rotated: [prev rotated by `rows`, query] stacked per sample -> [bs * 2, Q, C]
    (the reference's permute -> rotate -> permute -> torch.stack([prev_bev, bev_query], 1).reshape(bs * 2, Q, C))."""
    return RotateStack.apply(prev, query, rows)


def future_matrices(metas, future_frames):
    """`_align_bev_coordnates`' operands for each future frame k = 1 .. future_frames with a queue of one previous
    frame (detectors/vidar.py:196-215, :339-363): (future2ref[k], ref_to_history) -> float64 [F, bs, 4, 4] each,
    where ref_to_history starts as the current frame's ref_lidar_to_cur_lidar and becomes ref2future[k] after
    roll-out k.  Their product, in fp32 on the device as the reference forms it, moves the target grid."""
    f2r, r2h = [], []
    ref_to_history = [np.asarray(m["ref_lidar_to_cur_lidar"], np.float64) for m in metas]
    for k in range(1, future_frames + 1):
        f2r.append([np.asarray(m["future2ref_lidar_transform"][k], np.float64) for m in metas])
        r2h.append(ref_to_history)
        ref_to_history = [np.asarray(m["ref2future_lidar_transform"][k], np.float64) for m in metas]
    shape = (future_frames, len(metas), 4, 4)
    return np.array(f2r).reshape(shape), np.array(r2h).reshape(shape)


def future_grids(matrices, bev_h, bev_w, pc_range):
    """One future frame's previous-frame reference points: the BEV grid's centres in metres (bev_grids_to_coordinates,
    z = 0, w = 1) times `matrices` [bs, 4, 4] (device fp32, row-vector convention), back to grids
    (bev_coords_to_grids) and to [0, 1] -> [bs, Q, 1, 2]."""
    from . import bev_geometry
    bs = matrices.shape[0]
    grids = bev_geometry.get_bev_grids(bev_h, bev_w, bs, device=matrices.device, dtype=matrices.dtype)   # [bs, Q, 2]
    coords = bev_geometry.bev_grids_to_coordinates(grids, pc_range)
    coords = torch.cat([coords, torch.ones_like(coords[..., :2])], -1)                         # [bs, Q, 4]
    aligned = torch.matmul(coords, matrices)[..., :2]
    aligned, _ = bev_geometry.bev_coords_to_grids(aligned, bev_h, bev_w, pc_range)
    return ((aligned + 1) / 2.0).unsqueeze(2)


def future_inputs(metas, future_frames, bev_h, bev_w, pc_range, device, dtype=torch.float32):
    """The future decoder's inputs for roll-outs k = 1 .. future_frames from the current frame's `metas`
    (detectors/vidar.py:319-363) -> [(future_can_bus [bs, 4] at CAN_BUS_DIMS, ref_points [bs, Q, 1, 2] = `future_grids`
    of `future_matrices`' product)], one per roll-out.  The host values go up in one pinned upload in `dtype`; the
    product is formed on the device in `dtype` (the model's fp32, as vidar.py:215 forms it)."""
    fcb = np.array([[m["future_can_bus"][k][list(CAN_BUS_DIMS)] for m in metas]
                    for k in range(1, future_frames + 1)], np.float64)               # [F, bs, 4]
    f2r, r2h = future_matrices(metas, future_frames)                                  # [F, bs, 4, 4] each
    host = upload(np.concatenate([fcb.reshape(-1), f2r.reshape(-1), r2h.reshape(-1)]), device, dtype)
    n4, n16 = fcb.size, f2r.size
    fcb, f2r, r2h = host[:n4].view(fcb.shape), host[n4:n4 + n16].view(f2r.shape), host[n4 + n16:].view(r2h.shape)
    mats = torch.matmul(f2r, r2h)
    return [(fcb[k], future_grids(mats[k], bev_h, bev_w, pc_range)) for k in range(future_frames)]
