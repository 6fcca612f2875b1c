"""The K = 1 nearest-neighbour search (csrc/knn.cu) and the stable counting sort (csrc/counting_sort.cuh) at training
sizes, against host oracles: the batched search (chamfer.knn_points) at D = 2, 3, 4 and the segmented search
(vidar_nn_segments_forward) with exact ties on split, tile and random boundaries, bit for bit; the sort through its
three users (ray_head.align_gt, ray_head.decode_clouds, the dense Chamfer loss) over many chunks and up to 64 keys.
Cases: tests/nn_sort_cases.py."""
import numpy as np
import pytest
import torch

from oracle import dense_chamfer_ref, eval_ref, knn_ref
from tests import nn_sort_cases as nc
from tests.test_dense_chamfer_gpu import _grad_ok
from vidar_b200 import _lib, chamfer, ray_head

pytestmark = pytest.mark.gpu
NN_MASKED, NN_EMPTY = -1, -2          # include/vidar_b200.h


def _sms(cuda):
    return torch.cuda.get_device_properties(cuda).multi_processor_count


def _same_bits(got, want, what):
    """fp32 arrays equal bit for bit, NaN where the other is NaN (any NaN payload)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=f"{what}: NaN rows")
    bad = np.nonzero(got[~nan].view(np.int32) != want[~nan].view(np.int32))[0]
    assert bad.size == 0, f"{what}: {bad.size} values differ, first {got[~nan][bad[:3]]} vs {want[~nan][bad[:3]]}"


def _close64(got, want, what):
    """1e-5 relative plus a 1e-6 * max floor."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got - want)
    assert (err <= 1e-5 * np.abs(want) + 1e-6 * np.abs(want).max()).all(), f"{what}: max err {err.max():.3e}"


# ------------------------------------------------------------------ batched search
@pytest.mark.parametrize("D", [2, 3, 4])
def test_knn_points_forward_and_backward_match_oracle(cuda, D):
    c = nc.knn_case(D, _sms(cuda))
    p1 = torch.from_numpy(c["p1"]).to(cuda).requires_grad_(True)
    p2 = torch.from_numpy(c["p2"]).to(cuda).requires_grad_(True)
    k = chamfer.knn_points(p1, p2, lengths1=torch.from_numpy(c["len1"]).to(cuda),
                           lengths2=torch.from_numpy(c["len2"]).to(cuda))
    want_d, want_i = knn_ref.nn(c["p1"], c["p2"], c["len1"], c["len2"])
    np.testing.assert_array_equal(k.idx[..., 0].cpu().numpy(), want_i)
    _same_bits(k.dists[..., 0].detach().cpu().numpy(), want_d, "dists")
    (k.dists[..., 0] * torch.from_numpy(c["grad"]).to(cuda)).sum().backward()
    g1, g2 = knn_ref.nn_backward(c["p1"], c["p2"], want_i, c["grad"], c["len1"], c["len2"])
    _close64(p1.grad.cpu().numpy(), g1, "grad_p1")
    _close64(p2.grad.cpu().numpy(), g2, "grad_p2")
    # padding: zero distance, index 0, zero gradient; 400 queries scattered onto candidate 5 of element 0
    for n, (L1, L2) in enumerate(zip(c["len1"], c["len2"])):
        end = L1 if L2 else 0
        assert not k.dists[n, end:].any() and not k.idx[n, end:].any() and not p1.grad[n, end:].any()
        assert not p2.grad[n, L2:].any()
    assert int((k.idx[0, :, 0] == 5).sum()) >= 400 and float(p2.grad[0, 5].abs().sum()) > 0


# ------------------------------------------------------------------ segmented search
def _segments_oracle(c):
    Pq = len(c["q"])
    dists = np.zeros(Pq, np.float32)
    idx = np.full(Pq, NN_MASKED, np.int64)
    for s in range(len(c["q_off"]) - 1):
        q0, q1, c0, c1 = c["q_off"][s], c["q_off"][s + 1], c["c_off"][s], c["c_off"][s + 1]
        if q1 == q0:
            continue
        live = c["q_mask"][q0:q1].astype(bool)
        kept = np.nonzero(c["c_mask"][c0:c1])[0]
        if kept.size == 0:
            idx[q0:q1][live] = NN_EMPTY
            continue
        d, i = knn_ref.nn(c["q"][None, q0:q1], c["c"][None, c0 + kept])
        idx[q0:q1] = np.where(live, kept[i[0]], NN_MASKED)
        dists[q0:q1] = np.where(live, d[0], 0)
    return dists, idx


def test_segmented_search_matches_oracle(cuda):
    c = nc.segments_case(_sms(cuda))
    t = {k: torch.from_numpy(c[k]).to(cuda) for k in ("q", "c", "q_off", "c_off", "q_mask", "c_mask")}
    Pq, S = len(c["q"]), len(c["q_off"]) - 1
    dists = torch.empty(Pq, dtype=torch.float32, device=cuda)
    idx = torch.empty(Pq, dtype=torch.int64, device=cuda)
    scratch = torch.empty(Pq, dtype=torch.int64, device=cuda)
    P = _lib.ptr
    _lib.check(_lib.lib().vidar_nn_segments_forward(
        P(t["q"]), P(t["c"]), P(t["q_off"]), P(t["c_off"]), P(t["q_mask"]), P(t["c_mask"]), P(dists), P(idx),
        P(scratch), S, Pq, c["max_q"], c["max_c"], _lib.stream_ptr(cuda)))
    want_d, want_i = _segments_oracle(c)
    got_i = idx.cpu().numpy()
    np.testing.assert_array_equal(got_i, want_i)
    _same_bits(dists.cpu().numpy(), want_d, "dists")
    # every outcome occurs: masked queries, live queries without a kept candidate (two ways), nearest indices
    assert (got_i == NN_MASKED).any() and (got_i >= 0).any()
    for s in (1, nc.ALL_MASKED):
        seg = got_i[c["q_off"][s]:c["q_off"][s + 1]]
        assert (seg == NN_EMPTY).any() and set(seg.tolist()) <= {NN_EMPTY, NN_MASKED}


# ------------------------------------------------------------------ counting sort: GT alignment
def _align_oracle(gt, mats, jobs, voxel):
    """Per (head frame i, sample b): for each slot v in order, the rows of frame jobs[i, v] in their order, as
    x' = ((x T0 + y T4) + z T8) + T12 and ray = ((x' - off) * scale) * cells in fp32; then NaN / -1 padding."""
    H, V = jobs.shape
    bs, M, Cg = gt.shape
    off, scale, cells = voxel[:3], voxel[3:6], voxel[6:9]
    rays = np.full((H * bs, M, 3), np.nan, np.float32)
    pts = np.full((H * bs, M, 3), np.nan, np.float32)
    tidx = np.full((H * bs, M), -1.0, np.float32)
    for i in range(H):
        for b in range(bs):
            s, row = i * bs + b, 0
            for v in range(V):
                if jobs[i, v] < 0:
                    continue
                sel = np.nonzero(gt[b, :, Cg - 1] == np.float32(jobs[i, v]))[0]
                T = mats[i * V + v, b, :, :3]
                x, y, z = (gt[b, sel, a][:, None] for a in range(3))
                xp = ((x * T[0] + y * T[1]) + z * T[2]) + T[3]
                n = len(sel)
                pts[s, row:row + n] = xp
                rays[s, row:row + n] = ((xp - off) * scale) * cells
                tidx[s, row:row + n] = v
                row += n
    return rays, tidx, pts


@pytest.mark.parametrize("name", list(nc.ALIGN_CASES))
def test_align_gt_equals_masked_statements(cuda, name):
    c = nc.align_case(name)
    rays, tindex, pts = ray_head.align_gt(torch.from_numpy(c["gt"]).to(cuda), torch.from_numpy(c["mats"]).to(cuda),
                                          c["jobs"], c["voxel"], with_points=True)
    want = _align_oracle(c["gt"], c["mats"], c["jobs"], c["voxel"])
    for got, ref, what in zip((rays, tindex, pts), want, ("rays", "tindex", "points")):
        _same_bits(got.cpu().numpy(), ref, what)


# ------------------------------------------------------------------ counting sort: evaluation cloud decode
@pytest.mark.parametrize("name", list(nc.DECODE_CASES))
def test_decode_clouds_matches_oracle(cuda, name):
    c = nc.decode_case(name)
    t = {k: torch.from_numpy(c[k]).to(cuda) for k in ("depth", "rays", "points", "tindex", "origin_vox", "origin")}
    pred, gt, off = ray_head.decode_clouds(t["depth"], t["rays"], t["points"], t["tindex"], t["origin_vox"],
                                           t["origin"], c["scale"], c["within_grid"], c["pc_range"])
    want_pred, want_gt, want_off = eval_ref.decode_clouds(**c)
    np.testing.assert_array_equal(off.cpu().numpy(), want_off)
    _same_bits(pred.cpu().numpy(), want_pred, "pred")
    _same_bits(gt.cpu().numpy(), want_gt, "gt")
    F = c["origin"].shape[1]
    assert np.isnan(want_pred[want_off[-2]:]).all() and want_off[-2] < want_off[-1]
    if F > 2:                                   # the frame of no row is an empty cloud
        assert all(want_off[b * F + F - 2] == want_off[b * F + F - 1] for b in range(c["depth"].shape[0]))


# ------------------------------------------------------------------ counting sort + segmented search: dense Chamfer
def _check_pairs(got, want):
    got = got.cpu().numpy()
    np.testing.assert_array_equal(got[:, [1, 3]], want[:, [1, 3]])
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want[:, [0, 2]])
    np.testing.assert_allclose(got[:, [0, 2]][ok], want[:, [0, 2]][ok], rtol=1e-12, atol=0)


DENSE = {"few_pairs_split": (1, 2, 12000), "many_pairs": (4, 4, 6000)}     # (bs, F, M)


@pytest.mark.parametrize("name", list(DENSE))
def test_dense_chamfer_loss_gradient_and_pairs_match_oracle(cuda, name):
    bs, F, M = DENSE[name]
    c = nc.dense_case(bs, F, M=M, sms=_sms(cuda))
    assert (c["splits"] >= 2) == (name == "few_pairs_split")      # the search splits only with few pairs
    fw = [1.0 + 0.25 * f for f in range(F)]
    ws = float(sum(fw))
    t = {k: torch.from_numpy(c[k]).to(cuda) for k in ("dist", "points", "origin", "gt", "gt_tindex")}
    dist = t.pop("dist").requires_grad_(True)
    loss, pairs = ray_head.dense_chamfer_loss(dist, t["points"], t["origin"], t["gt"], t["gt_tindex"], nc.DENSE_GRID,
                                              fw, ws, return_pairs=True)
    loss.backward()
    want, want_grad, want_pairs = dense_chamfer_ref.dense_chamfer(
        c["dist"], c["points"], c["origin"], c["gt"], c["gt_tindex"], nc.DENSE_GRID, fw, ws, return_pairs=True)
    assert abs(float(loss.detach()) - want) <= 1e-5 * abs(want), (float(loss), want)
    got_grad = dist.grad.cpu().numpy()
    assert _grad_ok(got_grad, want_grad), np.abs(got_grad - want_grad).max()
    _check_pairs(pairs, want_pairs)


def test_dense_chamfer_group_loss_matches_oracle(cuda):
    """Three groups (one per frame) over two GT samples, the pair (sample 1, frame 1) left out."""
    bs, F, R0 = 2, 3, 2500
    c = nc.dense_case(bs, F, R0=R0, M=9000, sms=_sms(cuda))
    tab = [(s, f, s * F + f, f) for s in range(bs) for f in range(F) if (s, f) != (1, 1)]
    rays = np.concatenate([np.arange(s * F * R0 + f * R0, s * F * R0 + (f + 1) * R0) for s, f, _, _ in tab])
    dist = c["dist"].reshape(-1)[rays]
    points = c["points"].reshape(-1, 3)[rays]
    origin = c["origin"].reshape(-1, 3)
    w = np.float32([0.5, 1.0, 1.5, 0.75, 1.25])
    norms = np.float32([2.0, 3.0, 5.0])
    d = torch.from_numpy(dist).to(cuda).requires_grad_(True)
    loss, pairs = ray_head.dense_chamfer_group_loss(
        d, torch.from_numpy(points).to(cuda), torch.from_numpy(origin).to(cuda), torch.from_numpy(c["gt"]).to(cuda),
        torch.from_numpy(c["gt_tindex"]).to(cuda), nc.DENSE_GRID, tab, w, norms, return_pairs=True)
    loss.sum().backward()
    want, want_grad, want_pairs = dense_chamfer_ref.dense_chamfer_groups(
        dist, points, origin, c["gt"], c["gt_tindex"], nc.DENSE_GRID, tab, w, norms)
    np.testing.assert_allclose(loss.detach().cpu().numpy(), want, rtol=1e-5)
    got_grad = d.grad.cpu().numpy()
    assert _grad_ok(got_grad, want_grad), np.abs(got_grad - want_grad).max()
    _check_pairs(pairs, want_pairs)
