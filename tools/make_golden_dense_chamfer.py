"""Golden vectors of the head's dense Chamfer term from the REFERENCE's own ViDARHeadBase.loss run on CPU here,
with use_ce_loss = use_dist_loss = False, for every case of tests/dense_chamfer_cases.py.

    python tools/make_golden_dense_chamfer.py          # writes tests/golden/dense_chamfer.npz

`_custom_gumbel_softmax_distance` is replaced by a function returning the case's `dist` as a leaf tensor, so the
reference itself yields `loss.dense_voxel` and its gradient in dist.  The reference runs in float64 (inputs and
voxel grids), so the fixture pins the fp64 oracle (oracle/dense_chamfer_ref.py) to 1e-10.  mmdet3d's `chamfer_distance` is the
restatement in tools/make_golden_head.py.  The inputs of the batched op (ray end points, origin / GT grids and
frame indices as the reference builds them) are captured from the same call and stored beside the results,
one `<case>/<name>` entry per array.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import dense_chamfer_cases as dc  # noqa: E402
from tools import ref_shim  # noqa: E402
from tools.make_golden_head import chamfer_distance  # noqa: E402


def reference_head():
    utils = ref_shim.install_e2e_utils()
    f3 = utils.get_bev_grids_3d
    utils.get_bev_grids_3d = lambda H, W, Z, bs=1, device="cpu", dtype=None: f3(H, W, Z, bs, "cpu", torch.float64)
    mod = ref_shim.load("dense_heads.vidar_head_base")
    mod.chamfer_distance = chamfer_distance
    mod.e2e_predictor_utils = utils
    head = object.__new__(mod.ViDARHeadBase)
    torch.nn.Module.__init__(head)
    return head


def run(head, name):
    c = dc.case(name)
    for k, v in dict(ray_grid_num=16, ray_grid_step=1.0, use_ce_loss=False, use_dist_loss=False, use_dense_loss=True,
                     dense_loss_weight=1.0, eval_within_grid=c["within"]).items():
        setattr(head, k, v)
    head.loss_weight = np.array(dc.LOSS_W)
    dist = c["dist"].double().requires_grad_(True)
    seen = {}

    def decode(embed, length):
        assert tuple(embed.shape[:2]) == tuple(dist.shape), (embed.shape, dist.shape)
        return dist
    head._custom_gumbel_softmax_distance = decode
    process = type(head)._process_gt_points.__get__(head)
    render = type(head).get_rendered_pcds.__get__(head)

    def process_gt(*a, **k):
        out = process(*a, **k)
        seen.update(gt=out[2], gt_tindex=out[4])
        return out

    def rendered(origin, points, tindex, gt_dist, pred_dist, pc_range):
        seen.update(origin=origin, points=points)
        return render(origin, points, tindex, gt_dist, pred_dist, pc_range)
    head._process_gt_points, head.get_rendered_pcds = process_gt, rendered
    pd = dict(next_bev_preds=c["preds"].double(), valid_frames=list(range(dc.FRAMES)))
    loss = head.loss(pd, [p.double() for p in c["gt_points"]], pred_frame_num=dc.FRAMES,
                     batched_origin_points=c["origin"].double(),
                     **dc.call_kw(c))["loss.dense_voxel"]
    loss.backward()
    rec = dict(dist=dist.detach(), grad_dist=dist.grad, loss=loss.detach(), **seen)
    rec = {k: v.detach().numpy() for k, v in rec.items()}
    rec["grid"] = np.array([c["bev_w"], c["bev_h"], c["z"]])
    rec["pc_range"] = np.array(c["pc_range"], np.float64)
    rec["within"] = np.array(c["within"])
    print(f"{name}: loss {float(loss):.6g}, |grad| {float(dist.grad.abs().max()):.3g}, "
          f"{int((dist.grad != 0).sum())} rays with gradient")
    return rec


def main():
    head = reference_head()
    out = {}
    for name in dc.NAMES:
        for k, v in run(head, name).items():
            out[f"{name}/{k}"] = v
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "dense_chamfer.npz"), **out)


if __name__ == "__main__":
    main()
