"""Chamfer distance / nearest-neighbour op, H100-native (SURVEY.md 8(f) item 2).

Drop-in for the `chamferdist` package the reference builds from
third_lib/chamfer_dist/chamferdist: `knn_points` (K = 1 only -- the only K ViDAR uses) and
`ChamferDistance` with the reference's forward signature and returns (chamfer.py:20-133); used by
`compute_chamfer_distance` (projects/mmdet3d_plugin/bevformer/utils/e2e_predictor_utils.py:163-183).
CUDA tensors only.
"""
import warnings
from collections import namedtuple

import torch
from torch.autograd.function import once_differentiable

from . import _lib

_KNN = namedtuple("KNN", "dists idx knn")


class _knn_points(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p1, p2, lengths1, lengths2):
        _lib.require_cuda(p1=p1.contiguous(), p2=p2.contiguous())
        p1, p2 = p1.float().contiguous(), p2.float().contiguous()
        N, P1, D = p1.shape
        P2 = p2.shape[1]
        lengths1 = lengths1.to(torch.int64).contiguous()
        lengths2 = lengths2.to(torch.int64).contiguous()
        dists = torch.zeros((N, P1, 1), dtype=torch.float32, device=p1.device)
        idx = torch.zeros((N, P1, 1), dtype=torch.int64, device=p1.device)
        if P1 > 0 and P2 > 0:
            scratch = torch.empty((N, P1), dtype=torch.int64, device=p1.device)
            with torch.cuda.device(p1.device):
                _lib.check(_lib.lib().vidar_nn_forward(
                    _lib.ptr(p1), _lib.ptr(p2), _lib.ptr(lengths1), _lib.ptr(lengths2), _lib.ptr(dists),
                    _lib.ptr(idx), _lib.ptr(scratch), N, P1, P2, D, _lib.stream_ptr(p1.device)))
        ctx.save_for_backward(p1, p2, lengths1, lengths2, idx)
        ctx.mark_non_differentiable(idx)
        return dists, idx

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_dists, grad_idx):
        p1, p2, lengths1, lengths2, idx = ctx.saved_tensors
        N, P1, D = p1.shape
        P2 = p2.shape[1]
        grad_p1 = torch.zeros_like(p1)
        grad_p2 = torch.zeros_like(p2)
        if P1 > 0 and P2 > 0:
            g = grad_dists.float().contiguous()
            with torch.cuda.device(p1.device):
                _lib.check(_lib.lib().vidar_nn_backward(
                    _lib.ptr(p1), _lib.ptr(p2), _lib.ptr(lengths1), _lib.ptr(lengths2), _lib.ptr(idx), _lib.ptr(g),
                    _lib.ptr(grad_p1), _lib.ptr(grad_p2), N, P1, P2, D, _lib.stream_ptr(p1.device)))
        return grad_p1, grad_p2, None, None


def knn_points(p1, p2, lengths1=None, lengths2=None, K=1, version=-1, return_nn=False, return_sorted=True):
    """chamfer.py `knn_points` restricted to K = 1: -> KNN(dists [N,P1,1], idx [N,P1,1], knn)."""
    if K != 1:
        raise NotImplementedError("vidar_b200.chamfer.knn_points supports K = 1 (nearest neighbour) only")
    if p1.shape[0] != p2.shape[0]:
        raise ValueError("pts1 and pts2 must have the same batch dimension.")
    if p1.shape[2] != p2.shape[2]:
        raise ValueError("pts1 and pts2 must have the same point dimension.")
    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    if lengths1 is None:
        lengths1 = torch.full((N,), P1, dtype=torch.int64, device=p1.device)
    if lengths2 is None:
        lengths2 = torch.full((N,), P2, dtype=torch.int64, device=p1.device)
    dists, idx = _knn_points.apply(p1, p2, lengths1, lengths2)
    nn = None
    if return_nn:
        nn = p2[torch.arange(N, device=p1.device)[:, None, None], idx]       # [N, P1, 1, D]
    return _KNN(dists=dists, idx=idx, knn=nn)


class ChamferDistance(torch.nn.Module):
    """chamfer.py:20-133: same arguments, same returns."""

    def forward(self, source_cloud, target_cloud, bidirectional=False, reverse=False, reduction="mean"):
        if not isinstance(source_cloud, torch.Tensor) or not isinstance(target_cloud, torch.Tensor):
            raise TypeError("Expected input type torch.Tensor.")
        if source_cloud.device != target_cloud.device:
            raise ValueError("Source and target clouds must be on the same device. "
                             f"Got {source_cloud.device} and {target_cloud.device}.")
        bs, ls, ds = source_cloud.shape
        bt, lt, dt = target_cloud.shape
        if bs != bt:
            raise ValueError("Source and target pointclouds must have the same batchsize.")
        if ds != dt:
            raise ValueError("Source and target pointclouds must have the same dimensionality.")
        if bidirectional and reverse:
            warnings.warn("Both bidirectional and reverse set to True. bidirectional behavior takes precedence.")
        if reduction != "sum" and reduction != "mean" and reduction is not None:
            raise ValueError('Reduction must either be "sum" or "mean" or None.')
        len_s = torch.full((bs,), ls, dtype=torch.long, device=source_cloud.device)
        len_t = torch.full((bt,), lt, dtype=torch.long, device=target_cloud.device)
        src = knn_points(source_cloud, target_cloud, lengths1=len_s, lengths2=len_t, K=1)
        fwd_dist, fwd_idx = src.dists[..., 0], src.idx[..., 0]
        cham_f = fwd_dist.sum(1)
        cham_b = bwd_dist = bwd_idx = None
        if reverse or bidirectional:
            tgt = knn_points(target_cloud, source_cloud, lengths1=len_t, lengths2=len_s, K=1)
            bwd_dist, bwd_idx = tgt.dists[..., 0], tgt.idx[..., 0]
            cham_b = bwd_dist.sum(1)
        if reduction == "sum":
            cham_f = cham_f.sum()
            cham_b = cham_b.sum() if cham_b is not None else None
        elif reduction == "mean":
            cham_f = cham_f.mean()
            cham_b = cham_b.mean() if cham_b is not None else None
        if bidirectional:
            return cham_f, cham_b, (fwd_dist, fwd_idx, bwd_dist, bwd_idx)
        if reverse:
            return cham_b, (bwd_dist, bwd_idx)
        return cham_f, (fwd_dist, fwd_idx)


def compute_chamfer_distance(pred_pcd, gt_pcd):
    """bevformer/utils/e2e_predictor_utils.py:165-171."""
    loss_src, loss_dst, _ = ChamferDistance()(pred_pcd[None, ...], gt_pcd[None, ...], bidirectional=True, reduction="sum")
    return ((loss_src / pred_pcd.shape[0]) + (loss_dst / gt_pcd.shape[0])) / 2.0
