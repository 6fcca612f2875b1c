"""Argument validation of ViDARRayHeadV1 and of the alignment / grouped Chamfer entry points; runs without a GPU
(every check fires before anything touches the device)."""
import ctypes

import numpy as np
import pytest
import torch

from vidar_b200 import _lib, ray_head
from vidar_b200.head import ViDARRayHeadV1


def test_per_frame_loss_weight_must_cover_every_head_frame():
    with pytest.raises(ValueError, match="per_frame_loss_weight"):
        ViDARRayHeadV1(history_queue_length=4, pred_history_frame_num=3, pred_future_frame_num=1,
                       per_frame_loss_weight=(1.0, 1.0), loss_weight=[[1.0]])
    head = ViDARRayHeadV1(history_queue_length=4, pred_history_frame_num=1, pred_future_frame_num=1,
                          per_frame_loss_weight=(0.5, 1.0, 1.5), loss_weight=[[1.0], [0.0]])
    assert head.pred_frame_num == 3 and head.fuse_head_frames


def test_align_gt_rejects_bad_arguments():
    gt = torch.zeros(2, 10, 5)
    mats = torch.zeros(6, 2, 4, 4)
    vox = [0.0] * 9
    cases = [
        (dict(jobs=[1, 2, 3]), "jobs"),
        (dict(gt=torch.zeros(2, 10, 3)), "gt must be"),
        (dict(gt=gt.double()), "gt must be"),
        (dict(mats=torch.zeros(6, 1, 4, 4)), "mats must be"),
        (dict(voxel=[0.0] * 6), "voxel"),
        ({}, "CUDA"),
    ]
    for kw, needle in cases:
        args = dict(gt=gt, mats=mats, jobs=[[1, 2, 3], [2, 3, 4]], voxel=vox)
        args.update(kw)
        with pytest.raises(RuntimeError, match=needle):
            ray_head.align_gt(**args)


def test_dense_chamfer_group_loss_rejects_bad_tables():
    R0, M = 4, 6
    base = dict(dist=torch.zeros(2 * R0), points=torch.zeros(2 * R0, 3), origin=torch.zeros(4, 3),
                gt=torch.zeros(2, M, 3), gt_tindex=torch.zeros(2, M), grid=(8, 8, 4),
                pairs=[(0, 0, 0, 0), (1, 1, 3, 1)], pair_weights=[1.0, 1.0], group_norms=[1.0, 2.0])
    cases = [
        (dict(pairs=[(1, 1, 3, 1), (0, 0, 0, 0)]), "increasing"),
        (dict(pairs=[(0, 1, 0, 0), (0, 1, 3, 1)]), "increasing"),
        (dict(pairs=[(0, 0, 0, 0), (2, 1, 3, 1)]), "increasing"),
        (dict(pairs=[(0, 0, 0, 0), (1, 1, 4, 1)]), "out of range"),
        (dict(pairs=[(0, 0, 0, 0), (1, 1, 3, 2)]), "out of range"),
        (dict(pair_weights=[1.0]), "pairs"),
        (dict(dist=torch.zeros(2 * R0 + 1)), "dist must be"),
        (dict(gt_tindex=torch.zeros(2, M + 1)), "gt_tindex"),
        (dict(points=torch.zeros(2 * R0, 2)), "points"),
        (dict(dist=torch.zeros(2 * R0).double()), "float32"),
        ({}, "CUDA"),
    ]
    for kw, needle in cases:
        args = dict(base)
        args.update(kw)
        with pytest.raises(RuntimeError, match=needle):
            ray_head.dense_chamfer_group_loss(**args)


def test_c_entry_points_reject_bad_arguments():
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    jobs = ctypes.cast((ctypes.c_int32 * 8)(*range(8)), ctypes.c_void_p)
    vox = ctypes.cast((ctypes.c_float * 9)(*([0.0] * 9)), ctypes.c_void_p)
    rng = ctypes.cast((ctypes.c_float * 6)(0, 0, 0, 1, 1, 1), ctypes.c_void_p)

    def align(bs=1, M=100, Cg=5, H=2, V=4, ptr=X, jobs=jobs, vox=vox):
        return L.vidar_head_align_gt(X, X, jobs, vox, ptr, X, N, bs, M, Cg, H, V, N)

    def fwd(P=4, groups=2, R0=40, Sg=2, Fg=2, M=100, W=16, ptr=X, gt=X, pc=rng):
        return L.vidar_dense_chamfer_groups_forward(ptr, X, X, gt, gt, X, X, X, X, pc, X, X, X, X, X, X, X, X, X, P,
                                                    groups, R0, Sg, Fg, M, W, 16, 8, 0, N)

    def bwd(P=4, groups=2, R0=40, Sg=2, Fg=2, M=100, ptr=X):
        return L.vidar_dense_chamfer_groups_backward(X, X, X, X, X, X, X, X, X, X, X, X, X, ptr, P, groups, R0, Sg,
                                                     Fg, M, N)

    cases = [
        (align, dict(bs=0), b"bad sizes"), (align, dict(M=-1), b"bad sizes"), (align, dict(Cg=3), b"bad sizes"),
        (align, dict(V=65), b"bad sizes"), (align, dict(H=65, V=4), b"bad sizes"),
        (align, dict(bs=40000), b"segments"), (align, dict(jobs=N), b"null host table"),
        (align, dict(vox=N), b"null host table"), (align, dict(ptr=N), b"null pointer"),
        (fwd, dict(P=0), b"bad sizes"), (fwd, dict(groups=0), b"bad sizes"), (fwd, dict(Fg=65), b"bad sizes"),
        (fwd, dict(P=40000), b"pairs"), (fwd, dict(R0=1 << 30), b"rows"), (fwd, dict(W=0), b"bad grid"),
        (fwd, dict(R0=0), b"bad sizes"), (fwd, dict(M=-1), b"bad sizes"), (fwd, dict(pc=N), b"null pc_range"),
        (fwd, dict(ptr=N), b"null pointer"), (fwd, dict(gt=N), b"null gt buffer"),
        (bwd, dict(Sg=0), b"bad sizes"), (bwd, dict(ptr=N), b"null pointer"),
    ]
    for fn, kw, needle in cases:
        rc = fn(**kw)
        assert rc == 1, (kw, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (kw, L.vidar_last_error())
    # no gt rows is a valid size (every pair is then skipped); it fails only on the null output pointer here
    assert fwd(M=0, gt=N, ptr=N) == 1 and b"null pointer" in L.vidar_last_error()
