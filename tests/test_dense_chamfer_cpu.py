"""The head's dense Chamfer term without a GPU: the fp64 oracle against goldens made by the reference's own
ViDARHeadBase.loss (tools/make_golden_dense_chamfer.py), and argument validation of ray_head.dense_chamfer_loss."""
import os

import numpy as np
import pytest

from oracle import dense_chamfer_ref
from tests import dense_chamfer_cases as dc

GOLD = os.path.join(os.path.dirname(__file__), "golden", "dense_chamfer.npz")


def golden_case(g, name):
    """-> (arguments of ray_head.dense_chamfer_loss as numpy arrays / host values, loss, grad_dist)."""
    e = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    lw = np.array(dc.LOSS_W)
    args = dict(dist=e["dist"], points=e["points"], origin=e["origin"], gt=e["gt"], gt_tindex=e["gt_tindex"],
                grid=tuple(int(v) for v in e["grid"]), frame_weights=[float(w) for w in lw[:dc.FRAMES, 0]],
                weight_sum=float(lw.sum()), eval_within_grid=bool(e["within"]), pc_range=[float(v) for v in e["pc_range"]])
    return args, float(e["loss"]), e["grad_dist"]


@pytest.mark.parametrize("name", dc.NAMES)
def test_oracle_matches_reference_golden(name):
    g = np.load(GOLD)
    args, loss, grad = golden_case(g, name)
    got_loss, got_grad = dense_chamfer_ref.dense_chamfer(**args)
    assert abs(got_loss - loss) <= 1e-10 * abs(loss), (got_loss, loss)
    assert np.abs(got_grad - grad).max() <= 1e-10 * np.abs(grad).max()
    assert np.count_nonzero(grad) > 0


def test_cases_cover_what_they_are_named_for():
    g = np.load(GOLD)
    W = int(g["faces/grid"][0])
    gt, t = g["faces/gt"][0], g["faces/gt_tindex"][0]
    assert ((gt[:, 0] == 0) & (t >= 0)).sum() > 0 and ((gt[:, 0] == W - 1) & (t >= 0)).sum() > 0
    gt, t = g["gt_outside/gt"][0], g["gt_outside/gt_tindex"][0]
    assert (t == 1).sum() > 0 and (gt[t == 1, 0] >= W - 1).all()
    assert (g["dist_zero/dist"] == 0).mean() > 0.2 and (g["dist_zero/grad_dist"][g["dist_zero/dist"] == 0] == 0).all()
    assert bool(g["within_grid/within"])
    t = g["bs2_ragged/gt_tindex"]
    assert t.shape[0] == 2 and (t[0] >= 0).sum() > 10 * (t[1] >= 0).sum()
    # ties: repeated GT rows, and pred points that coincide (collinear rays of equal length)
    gt = g["ties/gt"][0]
    assert len(np.unique(gt[np.isfinite(gt).all(1)], axis=0)) < np.isfinite(gt).all(1).sum()
    R0 = g["ties/dist"].shape[1] // dc.FRAMES
    pts, o = g["ties/points"][0, :R0], g["ties/origin"][0, 0]
    r = pts - o
    live = np.linalg.norm(r, axis=1) > 0
    u = r[live] / np.linalg.norm(r[live], axis=1, keepdims=True)
    assert len(np.unique(u.round(12), axis=0)) < live.sum()


def test_dense_chamfer_loss_rejects_bad_arguments():
    """dense_chamfer_loss's own checks fire before anything touches the device (a GPU-less host can run this)."""
    import torch

    from vidar_b200 import ray_head
    bs, F, R0, M = 2, 3, 4, 6
    base = dict(dist=torch.zeros(bs, F * R0), points=torch.zeros(bs, F * R0, 3), origin=torch.zeros(bs, F, 3),
                gt=torch.zeros(bs, M, 3), gt_tindex=torch.zeros(bs, M), grid=(8, 8, 4), frame_weights=[1.0] * F,
                weight_sum=float(F))
    cases = [
        (dict(dist=torch.zeros(bs, F * R0 + 1)), "dist must be"),
        (dict(dist=torch.zeros(bs * F * R0)), "dist must be"),
        (dict(frame_weights=[]), "dist must be"),
        (dict(origin=torch.zeros(bs, F - 1, 3)), "origin"),
        (dict(points=torch.zeros(bs, F * R0, 2)), "points"),
        (dict(gt_tindex=torch.zeros(bs, M + 1)), "gt_tindex"),
        (dict(gt=torch.zeros(bs, M, 3).double(), gt_tindex=torch.zeros(bs, M).double()), "gt must be float32"),
        (dict(eval_within_grid=True), "pc_range"),
        ({}, "CUDA"),
    ]
    for kw, needle in cases:
        args = dict(base)
        args.update(kw)
        with pytest.raises(RuntimeError, match=needle):
            ray_head.dense_chamfer_loss(**args)
