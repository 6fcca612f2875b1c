"""ViDAR's evaluation metrics on the GPU (csrc/eval_metrics.cu over the segmented NN of csrc/knn.cu).

Drop-ins for the metric code of `forward_test`:
  compute_chamfer_distance_inner  utils/e2e_predictor_utils.py:173-183   same arguments / returns
  compute_ray_errors              utils/eval_utils.py:185-225             same arguments / returns
  frame_metrics                   detectors/vidar.py:452-497              the per-frame `ret_dict`
  summarize                       datasets/nuscenes_vidar_dataset_template.py:176-191 (evaluate's arithmetic)

frame_metrics scores every (sample, frame) pair of a batch in five kernel launches, whatever the batch size
and frame count, and copies one [bs * F, 8] float64 tensor to the host at the end.  Failures the reference
raises surface with the same exception types: a degenerate ray (RuntimeError), a clamped ray that never
touches the volume (AssertionError); gt points kept with no pred point kept, where the reference fails with an
IndexError, raise ValueError naming the (sample, frame).  CUDA tensors only.  `metrics_flat` is the same pass over
clouds already laid out flat with device offsets (the head's batched `evaluate` builds them on the device).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

# eval_utils.py reports at most these flags per cloud (include/vidar_b200.h VIDAR_EVAL_*)
GT_DEGENERATE, GT_OUTSIDE, INTERP_DEGENERATE, INTERP_OUTSIDE, NO_PRED = 1, 2, 4, 8, 16
FIELDS = 8      # sum l1, sum absrel, count, sum forward d, pred inside, sum backward d, gt inside, flags
DEFAULT_PC_RANGE = (-51.2, -51.2, -5.0, 51.2, 51.2, 3.0)


def _check_cloud(name, t):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must be [P, 3], got {tuple(t.shape)}")


def _device_offsets(sizes, device):
    """Exclusive prefix sums of host-known sizes, copied to the device without a host sync."""
    off = np.zeros(len(sizes) + 1, np.int64)
    np.cumsum(sizes, out=off[1:])
    host = torch.from_numpy(off).pin_memory()
    return host.to(device, non_blocking=True), int(off[-1])


def metrics_device(preds, gts, origins, pc_range=DEFAULT_PC_RANGE, rays=False):
    """Device part of the metrics of N = len(preds) (pred, gt, origin) triples.

    preds, gts: sequences of CUDA [P, 3] tensors; origins: CUDA [N, 3].  Launches only (no host sync).
    Returns a dict of device tensors: `out` [N, 8] float64 (FIELDS), and the intermediates -- `idx` / `dists`
    of the three searches over the query layout of vidar_eval_prologue, `q_mask`, `rays` [Pg, 9] (interpolated
    point, clamped gt, clamped interpolated point, when rays=True) -- plus the host-known sizes."""
    N = len(preds)
    if N == 0 or len(gts) != N:
        raise ValueError(f"need as many gt clouds as pred clouds (got {len(preds)} and {len(gts)}), at least one")
    for n in range(N):
        _check_cloud(f"pred_pcd[{n}]", preds[n])
        _check_cloud(f"gt_pcd[{n}]", gts[n])
    if not isinstance(origins, torch.Tensor) or not origins.is_cuda:
        raise RuntimeError("origin must be a CUDA tensor")
    dev = preds[0].device
    origin = origins.reshape(N, 3).to(torch.float32).contiguous()
    pred = torch.cat([p.to(torch.float32) for p in preds]).contiguous()
    gt = torch.cat([g.to(torch.float32) for g in gts]).contiguous()
    psz = [int(p.shape[0]) for p in preds]
    gsz = [int(g.shape[0]) for g in gts]
    offs, _ = _device_offsets(psz + gsz, dev)          # one copy: [pred_off | gt_off shifted by Pp]
    Pp = sum(psz)
    r = metrics_flat(pred, gt, origin, offs[: N + 1], offs[N:] - Pp, max(psz + gsz), pc_range, rays)
    return dict(r, pred_sizes=psz, gt_sizes=gsz)


def metrics_flat(pred, gt, origin, pred_off, gt_off, max_len, pc_range=DEFAULT_PC_RANGE, rays=False):
    """metrics_device once the clouds are flat: pred [Pp, 3], gt [Pg, 3], origin [N, 3] (float32, contiguous, CUDA),
    pred_off / gt_off [N + 1] int64 on the device (cloud n at rows [off[n], off[n+1]), the clouds tiling [0, Pp) and
    [0, Pg)), max_len a host bound of every cloud's size (a cloud of masked points only may be longer).  Four library
    calls, no host sync; returns the dict of metrics_device without the sizes."""
    N = int(origin.shape[0])
    dev = pred.device
    Pp, Pg = int(pred.shape[0]), int(gt.shape[0])
    Pq = Pp + 2 * Pg
    qbuf = torch.empty((Pq, 3), dtype=torch.float32, device=dev)
    cbuf = torch.empty((Pg + 2 * Pp, 3), dtype=torch.float32, device=dev)
    q_mask = torch.empty(Pq, dtype=torch.uint8, device=dev)
    c_mask = torch.empty(Pg + 2 * Pp, dtype=torch.uint8, device=dev)
    seg_off = torch.empty((2, 3 * N + 1), dtype=torch.int64, device=dev)
    dists = torch.empty(Pq, dtype=torch.float32, device=dev)
    idx = torch.empty(Pq, dtype=torch.int64, device=dev)
    scratch = torch.empty(Pq, dtype=torch.int64, device=dev)
    nbx = (max_len + 255) // 256
    partials = torch.empty(max(3 * N * nbx * 4, 1), dtype=torch.float64, device=dev)
    out = torch.empty((N, FIELDS), dtype=torch.float64, device=dev)
    ray_buf = torch.empty((Pg, 9), dtype=torch.float32, device=dev) if rays else None
    rng = (C.c_float * 6)(*[float(v) for v in pc_range])
    L = _lib.lib()
    st = _lib.stream_ptr(dev)
    P = _lib.ptr
    with torch.cuda.device(dev):
        _lib.check(L.vidar_eval_prologue(P(pred), P(gt), P(origin), P(pred_off), P(gt_off), C.cast(rng, C.c_void_p), P(qbuf), P(cbuf),
                                         P(q_mask), P(c_mask), P(seg_off[0]), P(seg_off[1]), N, Pp, Pg, st))
        _lib.check(L.vidar_nn_segments_forward(P(qbuf), P(cbuf), P(seg_off[0]), P(seg_off[1]), P(q_mask),
                                               P(c_mask), P(dists), P(idx), P(scratch), 3 * N, Pq, max_len,
                                               max_len, st))
        _lib.check(L.vidar_eval_metrics(P(pred), P(gt), P(origin), P(pred_off), P(gt_off), P(seg_off[0]),
                                        P(q_mask), P(dists), P(idx), P(partials), P(out), P(ray_buf), N, max_len,
                                        st))
    return dict(out=out, idx=idx, dists=dists, q_mask=q_mask, rays=ray_buf)


def raise_for_flags(flags, where):
    """Raise what the reference raises for a cloud with these VIDAR_EVAL_* flags, in the reference's order:
    the NN lookup (IndexError there, ValueError here), then clamp(gt), then clamp(interpolated points)."""
    flags = int(flags)
    if flags & NO_PRED:
        raise ValueError(f"{where}: gt points are kept but no pred point is farther than 1e-2 from the origin")
    if flags & GT_DEGENERATE:
        raise RuntimeError(f"{where}: a gt ray outside PC_RANGE ends at its origin")
    if flags & GT_OUTSIDE:
        raise AssertionError(f"{where}: a clamped gt ray does not touch the volume")
    if flags & INTERP_DEGENERATE:
        raise RuntimeError(f"{where}: an interpolated ray outside PC_RANGE ends at its origin")
    if flags & INTERP_OUTSIDE:
        raise AssertionError(f"{where}: a clamped interpolated ray does not touch the volume")


def chamfer_value(row):
    """compute_chamfer_distance_inner from one host row of `out`."""
    if row[4] == 0 or row[6] == 0:
        return 0.0
    return float((row[3] / row[4] + row[5] / row[6]) / 2.0)


def ray_values(row):
    """compute_ray_errors' (l1, absrel) from one host row of `out`; nan when no gt point is kept."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.float64(row[0]) / row[2]), float(np.float64(row[1]) / row[2])


def compute_chamfer_distance_inner(pred_pcd, gt_pcd, pc_range):
    """e2e_predictor_utils.py:173-183: 0.0 when either cloud has no point inside pc_range, else the Chamfer
    distance of the inside points as a 0-dim float32 tensor on their device."""
    _check_cloud("pred_pcd", pred_pcd)
    _check_cloud("gt_pcd", gt_pcd)
    origin = torch.zeros((1, 3), dtype=torch.float32, device=pred_pcd.device)
    row = metrics_device([pred_pcd], [gt_pcd], origin, pc_range)["out"][0].cpu().numpy()
    v = chamfer_value(row)
    if v == 0.0 and (row[4] == 0 or row[6] == 0):
        return 0.0
    return torch.tensor(v, dtype=torch.float32, device=pred_pcd.device)


def compute_ray_errors(pred_pcd, gt_pcd, origin, device=None, return_interpolated_pcd=False):
    """eval_utils.py:185-225 on CUDA tensors: (l1, absrel) as numpy.float32, or the interpolated points of the
    kept gt points ([count, 3] float32 numpy array) when return_interpolated_pcd.  `device` is accepted for
    signature compatibility; the work runs on the tensors' device."""
    _check_cloud("pred_pcd", pred_pcd)
    _check_cloud("gt_pcd", gt_pcd)
    if not isinstance(origin, torch.Tensor) or not origin.is_cuda:
        raise RuntimeError("origin must be a CUDA tensor")
    r = metrics_device([pred_pcd], [gt_pcd], origin.reshape(1, 3), rays=return_interpolated_pcd)
    row = r["out"][0].cpu().numpy()
    if return_interpolated_pcd:
        if int(row[7]) & NO_PRED:
            raise_for_flags(NO_PRED, "compute_ray_errors")
        Pp, Pg = r["pred_sizes"][0], r["gt_sizes"][0]
        kept = r["q_mask"][Pp + Pg:].bool()
        return r["rays"][kept, :3].cpu().numpy()
    raise_for_flags(row[7], "compute_ray_errors")
    l1, absrel = ray_values(row)
    return np.float32(l1), np.float32(absrel)


def frame_metrics_device(pred_pcds, gt_pcds, origin, pc_range):
    """Device part of frame_metrics: [bs * F, 8] float64 (row b * F + f), no host sync."""
    bs = len(pred_pcds)
    F = len(pred_pcds[0]) if bs else 0
    if bs == 0 or F == 0 or len(gt_pcds) != bs or any(len(p) != F or len(g) != F for p, g in zip(pred_pcds, gt_pcds)):
        raise ValueError("pred_pcds / gt_pcds must both be [bs][F] lists of clouds with bs, F >= 1")
    if tuple(origin.shape) != (bs, F, 3):
        raise ValueError(f"origin must be [bs, F, 3] = [{bs}, {F}, 3], got {tuple(origin.shape)}")
    preds = [pred_pcds[b][f] for b in range(bs) for f in range(F)]
    gts = [gt_pcds[b][f] for b in range(bs) for f in range(F)]
    return metrics_device(preds, gts, origin, pc_range)["out"]


def frame_metrics_host(out, bs, F, start_idx=0):
    """Host conversion of frame_metrics_device's result into vidar.py:452-497's ret_dict (Python numbers),
    raising the reference's exception of the first failing pair in its loop order (frame, then sample)."""
    out = out.cpu().numpy() if isinstance(out, torch.Tensor) else np.asarray(out)
    ret = {}
    for f in range(F):
        d = dict(count=0, chamfer_distance=0.0, l1_error=0.0, absrel_error=0.0)
        for b in range(bs):
            row = out[b * F + f]
            d["chamfer_distance"] += chamfer_value(row)
            raise_for_flags(row[7], f"sample {b}, frame {f + start_idx}")
            l1, absrel = ray_values(row)
            d["l1_error"] += l1
            d["absrel_error"] += absrel
            d["count"] += 1
        ret[f"frame.{f + start_idx}"] = d
    return ret


def frame_metrics(pred_pcds, gt_pcds, origin, pc_range, start_idx=0):
    """vidar.py:452-497: pred_pcds[b][f], gt_pcds[b][f] ([P, 3] CUDA tensors) and origin [bs, F, 3] as
    get_point_cloud_prediction returns them -> {f"frame.{f + start_idx}": {count, chamfer_distance,
    l1_error, absrel_error}}, each value summed over the batch in batch order."""
    out = frame_metrics_device(pred_pcds, gt_pcds, origin, pc_range)
    return frame_metrics_host(out, len(pred_pcds), len(pred_pcds[0]), start_idx)


def summarize(results):
    """The dataset's evaluate() (nuscenes_vidar_dataset_template.py:176-191): sum the per-sample ret_dicts
    key by key, then divide every metric of a frame by its count.  Host code; returns a new dict."""
    total = None
    for result in results:
        if total is None:
            total = {k: dict(v) for k, v in result.items()}
        else:
            for frame_k, frame_res in result.items():
                for k, v in frame_res.items():
                    total[frame_k][k] += v
    if total is None:
        return {}
    for frame_res in total.values():
        count = frame_res["count"]
        for k, v in frame_res.items():
            if k != "count":
                frame_res[k] = v / count
    return total
