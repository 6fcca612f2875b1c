"""The head's dense Chamfer term without a GPU: the fp64 oracle against goldens made by the reference's own
ViDARHeadBase.loss (tools/make_golden_dense_chamfer.py), and argument validation of the C entry points."""
import ctypes
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


def test_entry_points_reject_bad_arguments():
    """Sizes and pointers are checked before anything touches the device (a GPU-less host can run this)."""
    from vidar_b200 import _lib
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    w = ctypes.cast((ctypes.c_float * 4)(1, 1, 1, 1), ctypes.c_void_p)
    rng = ctypes.cast((ctypes.c_float * 6)(0, 0, 0, 1, 1, 1), ctypes.c_void_p)

    def fwd(bs=1, F=2, R0=40, To=2, M=100, W=16, H=16, Z=8, ptr=X, gt=X, weights=w, pc=rng):
        return L.vidar_dense_chamfer_forward(ptr, X, X, gt, gt, weights, pc, 2.0, X, X, X, X, X, X, X, X, X, bs, F,
                                             R0, To, M, W, H, Z, 0, N)

    def bwd(bs=1, F=2, R0=40, To=2, M=100, ptr=X, weights=w):
        return L.vidar_dense_chamfer_backward(X, X, X, X, X, X, X, X, X, weights, 2.0, X, ptr, bs, F, R0, To, M, N)

    cases = [
        (fwd, dict(bs=0), b"bad sizes"), (fwd, dict(F=0), b"bad sizes"), (fwd, dict(F=65), b"bad sizes"),
        (fwd, dict(R0=0), b"bad sizes"), (fwd, dict(To=1), b"bad sizes"), (fwd, dict(M=-1), b"bad sizes"),
        (fwd, dict(W=0), b"bad grid"), (fwd, dict(bs=20000), b"pairs"), (fwd, dict(R0=1 << 30), b"rows"),
        (fwd, dict(ptr=N), b"null pointer"), (fwd, dict(gt=N), b"null gt"), (fwd, dict(weights=N), b"null loss weights"),
        (fwd, dict(pc=N), b"null pc_range"),
        (bwd, dict(F=0), b"bad sizes"), (bwd, dict(To=1), b"bad sizes"), (bwd, dict(ptr=N), b"null pointer"),
        (bwd, dict(weights=N), b"null loss weights"),
    ]
    for fn, kw, needle in cases:
        rc = fn(**kw)
        assert rc == 1, (kw, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (kw, L.vidar_last_error())
    # no gt rows is a valid size (every pair is then skipped); it fails only on the null output pointer here
    assert fwd(M=0, gt=N, ptr=N) == 1 and b"null pointer" in L.vidar_last_error()
