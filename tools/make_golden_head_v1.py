"""Golden vectors for ViDARHeadV1 from the REFERENCE methods run on CPU here: ViDARHeadV1.loss (every
'frame.{idx}.{k}.loss' key and the gradient w.r.t. next_bev_preds) and get_point_cloud_prediction
(dense_heads/vidar_head_v1.py:94-252), for the cases of tests/head_v1_cases.py.

    python tools/make_golden_head_v1.py          # writes tests/golden/head_v1.npz

`chamfer_distance` and the e2e_predictor_utils helpers come from tools/make_golden_head.py / tools/ref_shim.py.
The Gumbel noise the reference draws (CPU generator, seed 11; one dense-term draw per head frame) is re-drawn here
in the same order and stored for the frames of non-zero weight (`head_v1_cases.weighted_frames`), so the GPU tests
feed the identical noise; the noise of zero-weight frames changes no loss and no gradient.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import head_v1_cases as hc  # noqa: E402
from tools import ref_shim  # noqa: E402
from tools.make_golden_head import chamfer_distance  # noqa: E402

SEED = 11


def make_head():
    utils = ref_shim.install_e2e_utils()
    f3 = utils.get_bev_grids_3d
    utils.get_bev_grids_3d = lambda H, W, Z, bs=1, device="cpu", dtype=torch.float: f3(H, W, Z, bs, "cpu", dtype)
    base = ref_shim.load("dense_heads.vidar_head_base")
    base.chamfer_distance = chamfer_distance
    base.e2e_predictor_utils = utils
    mod = ref_shim.load("dense_heads.vidar_head_v1")
    head = object.__new__(mod.ViDARHeadV1)
    torch.nn.Module.__init__(head)
    kw = dict(hc.HEAD_KW)
    for k in ("history_queue_length", "pred_history_frame_num", "pred_future_frame_num", "per_frame_loss_weight"):
        setattr(head, k, kw.pop(k))
    head.pred_frame_num = 1 + head.pred_history_frame_num + head.pred_future_frame_num
    for k, v in kw.items():
        setattr(head, k, v)
    head.loss_weight = np.array(hc.LOSS_W)
    return head


def main():
    head = make_head()
    rec, grads, draws = {}, {}, {}
    for name in hc.CASES:
        c = hc.case(name)
        preds = c["pred_dict"]["next_bev_preds"].clone().requires_grad_(True)
        pd = dict(c["pred_dict"], next_bev_preds=preds)
        shapes = []
        orig = head._custom_gumbel_softmax_distance
        head._custom_gumbel_softmax_distance = lambda e, l: (shapes.append(tuple(e.shape)), orig(e, l))[1]
        torch.manual_seed(SEED)
        losses = head.loss(pd, c["gt_points"], pred_frame_num=None, img_metas=c["img_metas"], **hc.CALL_KW)
        del head._custom_gumbel_softmax_distance
        sum(losses.values()).backward()
        for k, v in losses.items():
            rec[f"{name}/loss/{k}"] = v.detach().numpy()
        assert float(preds.grad[:, :-1].abs().sum()) == 0      # only the last intermediate output is supervised
        grads[name] = preds.grad[:, -1].numpy()
        torch.manual_seed(SEED)
        draws[name] = [(-torch.empty(shp).exponential_().log()).numpy() for shp in shapes]
        src = hc.SAME_DRAWS.get(name)
        if src is not None:
            # one copy in the golden: the same draws, and the source's gradient of the current head frame alone
            assert all(np.array_equal(a, b) for a, b in zip(draws[name], draws[src]))
            ref = np.zeros_like(grads[src])
            phf = hc.HEAD_KW["pred_history_frame_num"]
            ref[:, phf] = grads[src][:, phf]
            assert np.array_equal(grads[name], ref)
        else:
            rec[f"{name}/grad_preds_last"] = grads[name]
            V = len(c["pred_dict"]["valid_frames"])
            for idx, noise in enumerate(draws[name]):
                R0 = noise.shape[1] // V
                frames = hc.weighted_frames(name, idx)
                if frames:
                    rec[f"{name}/gumbel_dense_{idx}"] = np.concatenate(
                        [noise[:, t * R0:(t + 1) * R0] for t in frames], 1)
        print(name, {k: float(v) for k, v in losses.items()}, shapes)
        with torch.no_grad():
            dec = head.get_point_cloud_prediction(dict(c["pred_dict"]), c["gt_points"], img_metas=c["img_metas"],
                                                  **hc.CALL_KW)
        for key in ("pred_pcds", "gt_pcds"):
            for b in range(hc.BS):
                for t in range(len(c["pred_dict"]["valid_frames"])):
                    rec[f"{name}/{key}_{b}_{t}"] = dec[key][b][t].numpy()
        rec[f"{name}/origin"] = dec["origin"].numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "head_v1.npz"), **rec)


if __name__ == "__main__":
    main()
