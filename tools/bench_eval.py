"""Time ViDAR's evaluation metrics on one decode-sized sample: 7 frames x ~30 k points of the LiDAR pattern of
tests/eval_cases.py.

  batched   vidar_b200.evaluate.frame_metrics: five launches for all frames, one copy to the host
  per-pair  the path the reference takes (vidar.py:452-497): per frame, compute_chamfer_distance on the
            boolean-masked clouds (this package's CUDA Chamfer), then compute_ray_errors with numpy on the host
            around a device NN search (eval_utils.py:185-225, restated by oracle/eval_ref.py), with its syncs

Wall-clock time of each call ending in a device synchronise (both paths end on the host), and CUDA events around
the batched call in a run of their own as a cross-check; median of --reps after --warmup.  Prints one JSON line with
the card, its power limit and SM clock read in the same run.

    python tools/bench_eval.py [--points 30000] [--frames 7] [--reps 20] [--ref-reps 5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import eval_ref  # noqa: E402
from tests.eval_cases import PC_RANGE, frame  # noqa: E402
from tools.gpu_timing import card, event_ms, host_ms  # noqa: E402
from vidar_b200 import chamfer, evaluate  # noqa: E402


def per_pair(pred_pcds, gt_pcds, origin, dev):
    """vidar.py:452-497 for one sample, as the reference runs it."""
    res = {}
    cd_fn = chamfer.ChamferDistance()
    for f in range(len(pred_pcds)):
        p, g = pred_pcds[f], gt_pcds[f]
        pm, gm = evaluate_inside(p), evaluate_inside(g)
        ip, ig = p[pm], g[gm]                                            # host syncs, as in the reference
        cd = 0.0 if (pm.sum() == 0 or gm.sum() == 0) else chamfer.compute_chamfer_distance(ip, ig).item()
        pn, gn, o = p.cpu().numpy(), g.cpu().numpy(), origin[f].cpu().numpy()
        th_h, ph_h, d_h = eval_ref.spherical_projection(pn - o[None])
        th, ph, d = eval_ref.spherical_projection(gn - o[None])
        mh, m = d_h > np.float32(1e-2), d > np.float32(1e-2)
        ps = np.stack([th_h[mh], ph_h[mh], np.ones(int(mh.sum()), np.float32)], 1)
        gs = np.stack([th[m], ph[m], np.ones(int(m.sum()), np.float32)], 1)
        _, info = cd_fn(torch.from_numpy(ps[None]).to(dev), torch.from_numpy(gs[None]).to(dev), reverse=True)
        idx = info[1].cpu().numpy()[0]
        gt = gn[m]
        v = gt - o[None]
        interp = o[None] + d_h[mh][idx][:, None] * (v / np.sqrt((v * v).sum(1, keepdims=True)))
        go, gc, inv = eval_ref.clamp(gt, o)
        _, ic, _ = eval_ref.clamp(interp, o)
        keep = ~inv
        dc = np.sqrt(((gc[keep] - go[keep]) ** 2).sum(1))
        valid = dc > np.float32(0.01)
        l1 = np.sqrt(((gc[keep][valid] - ic[keep][valid]) ** 2).sum(1))
        res[f] = (cd, l1.sum() / len(gt), (l1 / dc[valid]).sum() / len(gt))
    return res


def evaluate_inside(p):
    lo = torch.tensor(PC_RANGE[:3], device=p.device)
    hi = torch.tensor(PC_RANGE[3:], device=p.device)
    return ((lo <= p) & (p <= hi)).all(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=30000)
    ap.add_argument("--frames", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval needs a CUDA device")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    frs = [frame(rng, a.points + 97 * f, np.array([0.3 * f, -0.2 * f, 1.8], np.float32)) for f in range(a.frames)]
    pred_pcds = [[torch.from_numpy(p).to(dev) for p, _, _ in frs]]
    gt_pcds = [[torch.from_numpy(g).to(dev) for _, g, _ in frs]]
    origin = torch.from_numpy(np.stack([o for _, _, o in frs]))[None].to(dev)

    def batched():
        return evaluate.frame_metrics(pred_pcds, gt_pcds, origin, PC_RANGE)

    def reference():
        return per_pair(pred_pcds[0], gt_pcds[0], origin[0], dev)

    t = host_ms(batched, a.reps, a.warmup)
    t_events = event_ms(batched, a.reps, a.warmup)
    got = batched()
    want = reference()                                         # also the reference's warm-up
    t_ref = host_ms(reference, a.ref_reps, 0)

    worst = 0.0
    for f in range(a.frames):
        g = got[f"frame.{f}"]
        for m, w in zip(("chamfer_distance", "l1_error", "absrel_error"), want[f]):
            worst = max(worst, abs(g[m] - float(w)) / max(abs(float(w)), 1e-30))
    pairs = sum(3 * len(p) * len(g) for p, g, _ in frs)       # candidates scanned by the three searches
    print(json.dumps(dict(
        metric="eval_frame_metrics", frames=a.frames, points=[len(g) for _, g, _ in frs],
        batched_ms=round(t, 3), batched_events_ms=round(t_events, 3), per_pair_ms=round(t_ref, 1),
        speedup=round(t_ref / t, 1), nn_pairs_per_s=float(f"{pairs / (t * 1e-3):.4g}"), reps=a.reps,
        ref_reps=a.ref_reps, max_rel_diff=worst, **card())))


if __name__ == "__main__":
    main()
