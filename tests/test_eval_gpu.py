"""ViDAR's evaluation metrics on the GPU (vidar_b200.evaluate): against goldens made by the reference's own
eval_utils.py, against the oracle at decode size, and the properties of the batched path."""
import math

import numpy as np
import pytest
import torch

from oracle import eval_ref
from tests.eval_cases import PC_RANGE, frame
from tests.test_eval_cpu import golden_frames, spherical_mismatches

pytestmark = pytest.mark.gpu


def _dev(cuda, frames):
    preds = [torch.from_numpy(p).to(cuda) for p, _, _ in frames]
    gts = [torch.from_numpy(g).to(cuda) for _, g, _ in frames]
    origins = torch.from_numpy(np.stack([o for _, _, o in frames])).to(cuda)
    return preds, gts, origins


def test_cuda_matches_reference_goldens(cuda):
    from vidar_b200 import evaluate
    g, frames = golden_frames()
    preds, gts, origins = _dev(cuda, frames)
    r = evaluate.metrics_device(preds, gts, origins, PC_RANGE, rays=True)     # every golden frame in one call
    out = r["out"].cpu().numpy()
    idx, q_mask, rays = r["idx"].cpu().numpy(), r["q_mask"].cpu().numpy().astype(bool), r["rays"].cpu().numpy()
    Pp, Pg = sum(r["pred_sizes"]), sum(r["gt_sizes"])
    total, differ, p0, g0 = 0, 0, 0, 0
    for k, (pred, gt, origin) in enumerate(frames):
        row = out[k]
        assert int(row[7]) == 0
        l1, absrel = evaluate.ray_values(row)
        np.testing.assert_allclose([l1, absrel], [g[f"l1_{k}"], g[f"absrel_{k}"]], rtol=1e-5, err_msg=f"frame {k}")
        np.testing.assert_allclose(evaluate.chamfer_value(row), g[f"chamfer_{k}"], rtol=1e-5, err_msg=f"frame {k}")
        P, G = len(pred), len(gt)
        kept = q_mask[Pp + Pg + g0:Pp + Pg + g0 + G]
        _, _, d_hat = eval_ref.spherical_projection(pred - origin[None])
        kept_hat = d_hat > np.float32(1e-2)
        compact = np.cumsum(kept_hat) - 1                             # raw index -> index among kept pred points
        raw = idx[Pp + Pg + g0:Pp + Pg + g0 + G][kept]
        assert (raw >= 0).all()
        bad = spherical_mismatches(g, k, pred, gt, origin, compact[raw])
        fr = rays[g0:g0 + G][kept]
        np.testing.assert_array_equal(fr[:, 3:6], g[f"clamped_gt_{k}"])
        np.testing.assert_array_equal(fr[~bad, 0:3], g[f"interp_{k}"][~bad])
        np.testing.assert_array_equal(fr[~bad, 6:9], g[f"clamped_interp_{k}"][~bad])
        total += len(bad)
        differ += int(bad.sum())
        p0, g0 = p0 + P, g0 + G
    print(f"NN differences explained by arctan2 rounding or near ties: {differ} of {total}")
    assert differ < 1e-3 * total


def _decode_batch(sizes, seed):
    rng = np.random.default_rng(seed)
    out = []
    for row in sizes:
        fr = []
        for n in row:
            o = np.array([rng.uniform(-3, 3), rng.uniform(-3, 3), 1.8], np.float32)
            if n == 0:
                fr.append((np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), o))
            elif n == 1:
                fr.append((o[None] + np.float32([[4.0, 3.0, -1.0]]), o[None] + np.float32([[8.0, 6.5, -1.5]]), o))
            else:
                fr.append(frame(rng, n, o))
        out.append(fr)
    return out


SIZES = [[30000, 29000, 0, 1, 3000, 28000, 500], [27000, 1, 30500, 0, 2000, 100, 31000]]
FULL_ORACLE = {(0, 0), (1, 6)}          # the 30 k pairs the oracle recomputes completely (its NN is numpy)


def test_cuda_matches_oracle_at_decode_size(cuda):
    from vidar_b200 import evaluate
    batch = _decode_batch(SIZES, seed=3)
    bs, F = len(batch), len(batch[0])
    pred_pcds = [[torch.from_numpy(batch[b][f][0]).to(cuda) for f in range(F)] for b in range(bs)]
    gt_pcds = [[torch.from_numpy(batch[b][f][1]).to(cuda) for f in range(F)] for b in range(bs)]
    origin = torch.from_numpy(np.stack([np.stack([batch[b][f][2] for f in range(F)]) for b in range(bs)])).to(cuda)
    out = evaluate.frame_metrics_device(pred_pcds, gt_pcds, origin, PC_RANGE).cpu().numpy()
    checked = 0
    for b in range(bs):
        for f in range(F):
            pred, gt, o = batch[b][f]
            row = out[b * F + f]
            assert int(row[7]) == 0, (b, f, row[7])
            if len(gt) > 3000 and (b, f) not in FULL_ORACLE:
                continue
            l1, absrel = eval_ref.compute_ray_errors(pred, gt, o)
            cd = eval_ref.compute_chamfer_distance_inner(pred, gt, PC_RANGE)
            got = evaluate.ray_values(row)
            if len(gt) == 0:
                assert math.isnan(got[0]) and math.isnan(l1) and evaluate.chamfer_value(row) == 0.0 == cd
                continue
            np.testing.assert_allclose(got, [l1, absrel], rtol=1e-5, err_msg=f"{(b, f)}")
            np.testing.assert_allclose(evaluate.chamfer_value(row), cd, rtol=1e-5, err_msg=f"{(b, f)}")
            checked += 1
    assert checked >= 8
    # every 30 k pair: the counts are exact, and a cloud scored alone gives the same row bit for bit
    for b, f in ((0, 1), (1, 2)):
        alone = evaluate.metrics_device([pred_pcds[b][f]], [gt_pcds[b][f]], origin[b, f][None], PC_RANGE)["out"]
        assert np.array_equal(alone.cpu().numpy()[0], out[b * F + f])


def test_frame_metrics_matches_per_pair_loop(cuda):
    from vidar_b200 import evaluate
    _, frames = golden_frames()
    for bs, F in ((1, 7), (2, 3)):
        fr = [[frames[(b * F + f) % len(frames)] for f in range(F)] for b in range(bs)]
        want = eval_ref.frame_metrics([[x[0] for x in r] for r in fr], [[x[1] for x in r] for r in fr],
                                      np.stack([np.stack([x[2] for x in r]) for r in fr]), PC_RANGE, start_idx=1)
        got = evaluate.frame_metrics([[torch.from_numpy(x[0]).to(cuda) for x in r] for r in fr],
                                     [[torch.from_numpy(x[1]).to(cuda) for x in r] for r in fr],
                                     torch.from_numpy(np.stack([np.stack([x[2] for x in r]) for r in fr])).to(cuda),
                                     PC_RANGE, start_idx=1)
        assert list(got) == list(want) == [f"frame.{f + 1}" for f in range(F)]
        for k in want:
            assert got[k]["count"] == want[k]["count"] == bs
            for m in ("chamfer_distance", "l1_error", "absrel_error"):
                assert isinstance(got[k][m], float)
                np.testing.assert_allclose(got[k][m], want[k][m], rtol=1e-5, err_msg=f"{bs} {k} {m}")


def test_single_pair_functions(cuda):
    from vidar_b200 import evaluate
    g, frames = golden_frames()
    pred, gt, o = frames[0]
    l1, absrel = evaluate.compute_ray_errors(torch.from_numpy(pred).to(cuda), torch.from_numpy(gt).to(cuda),
                                             torch.from_numpy(o).to(cuda), cuda)
    assert isinstance(l1, np.float32) and isinstance(absrel, np.float32)
    np.testing.assert_allclose([l1, absrel], [g["l1_0"], g["absrel_0"]], rtol=1e-5)
    interp = evaluate.compute_ray_errors(torch.from_numpy(pred).to(cuda), torch.from_numpy(gt).to(cuda),
                                         torch.from_numpy(o).to(cuda), return_interpolated_pcd=True)
    np.testing.assert_array_equal(interp, g["interp_0"])
    cd = evaluate.compute_chamfer_distance_inner(torch.from_numpy(pred).to(cuda), torch.from_numpy(gt).to(cuda),
                                                 PC_RANGE)
    assert cd.dtype == torch.float32 and cd.device.type == "cuda"
    np.testing.assert_allclose(cd.item(), g["chamfer_0"], rtol=1e-5)
    p6, g6, _ = frames[6]
    assert evaluate.compute_chamfer_distance_inner(torch.from_numpy(p6).to(cuda), torch.from_numpy(g6).to(cuda),
                                                   PC_RANGE) == 0.0
    with pytest.raises(RuntimeError, match="CUDA"):
        evaluate.compute_ray_errors(torch.from_numpy(pred), torch.from_numpy(gt), torch.from_numpy(o))


def test_failures_raise_the_reference_exception_types(cuda):
    from vidar_b200 import evaluate
    t = lambda a: torch.tensor(a, dtype=torch.float32, device=cuda)
    o = t([0.0, 0.0, 0.0])
    gt = t([[5.0, 1.0, 0.5]])
    with pytest.raises(ValueError):                                     # no pred point kept (IndexError there)
        evaluate.compute_ray_errors(t([[0.0, 0.0, 0.0], [1e-3, 0.0, 0.0]]), gt, o)
    with pytest.raises(RuntimeError):                                   # degenerate interpolated ray
        evaluate.compute_ray_errors(t([[1e6, 0.02, 0.0]]), t([[1e6 + 0.0625, 0.0, 0.0]]), t([1e6, 0.0, 0.0]))
    with pytest.raises(AssertionError):                                 # ray that never touches the volume
        evaluate.compute_ray_errors(t([[float("inf"), 3.0, 0.0]]), gt, o)
    # the batched path names the failing pair
    ok_p, ok_g = t([[4.0, 3.0, 0.0]]), t([[8.0, 6.0, 0.5]])
    with pytest.raises(ValueError, match="sample 1, frame 0"):
        evaluate.frame_metrics([[ok_p, ok_p], [t([[0.0, 0.0, 0.0]]), ok_p]], [[ok_g, ok_g], [ok_g, ok_g]],
                               torch.zeros(2, 2, 3, device=cuda), PC_RANGE)


def test_two_calls_are_bit_identical(cuda):
    from vidar_b200 import evaluate
    batch = _decode_batch([[6000, 5000, 1], [4000, 0, 7000]], seed=5)
    preds, gts, origins = _dev(cuda, [x for r in batch for x in r])
    a = evaluate.metrics_device(preds, gts, origins, PC_RANGE)["out"]
    b = evaluate.metrics_device(preds, gts, origins, PC_RANGE)["out"]
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_launch_count_is_independent_of_batch(cuda):
    from vidar_b200 import _lib, evaluate
    for bs in (1, 2):
        batch = _decode_batch([[2000, 1500, 1000]] * bs, seed=bs)
        pred_pcds = [[torch.from_numpy(x[0]).to(cuda) for x in r] for r in batch]
        gt_pcds = [[torch.from_numpy(x[1]).to(cuda) for x in r] for r in batch]
        origin = torch.from_numpy(np.stack([np.stack([x[2] for x in r]) for r in batch])).to(cuda)
        n0 = _lib.launch_count()
        evaluate.frame_metrics(pred_pcds, gt_pcds, origin, PC_RANGE)
        assert _lib.launch_count() - n0 == 5, bs


def test_device_part_has_no_host_sync(cuda):
    from vidar_b200 import evaluate
    batch = _decode_batch([[3000, 2000], [2500, 1]], seed=7)
    pred_pcds = [[torch.from_numpy(x[0]).to(cuda) for x in r] for r in batch]
    gt_pcds = [[torch.from_numpy(x[1]).to(cuda) for x in r] for r in batch]
    origin = torch.from_numpy(np.stack([np.stack([x[2] for x in r]) for r in batch])).to(cuda)
    evaluate.frame_metrics_device(pred_pcds, gt_pcds, origin, PC_RANGE)       # warm the allocators
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = evaluate.frame_metrics_device(pred_pcds, gt_pcds, origin, PC_RANGE)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    ret = evaluate.frame_metrics_host(out, 2, 2)
    assert ret["frame.1"]["count"] == 2 and math.isfinite(ret["frame.0"]["l1_error"])
