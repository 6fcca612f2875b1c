"""Golden vectors for ViDAR's evaluation metrics from the REFERENCE's own code run on CPU here:
utils/eval_utils.py imported unmodified (its `chamferdist` is the reference chamfer.py over the reference's CPU
KNN build oracle/_ref/ref_knn_cpu.so, as in tools/make_golden_knn.py), and compute_chamfer_distance_inner /
get_inside_mask / compute_chamfer_distance of utils/e2e_predictor_utils.py through ref_shim.load_functions (the
module JIT-compiles CUDA at import).  Inputs from tests/eval_cases.py.  Writes tests/golden/eval.npz.

    python tools/make_golden_eval.py
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle import build_ref  # noqa: E402
from tests.eval_cases import PC_RANGE, cases  # noqa: E402

CHAMFERDIST = "/root/reference/third_lib/chamfer_dist/chamferdist/chamferdist"
EVAL_UTILS = "/root/reference/projects/mmdet3d_plugin/bevformer/utils/eval_utils.py"


def _install_chamferdist():
    build_ref.build_knn_cpu()
    pkg = types.ModuleType("chamferdist")
    pkg._C = build_ref.load("ref_knn_cpu")
    pkg.__path__ = []
    sys.modules["chamferdist"] = pkg
    spec = importlib.util.spec_from_file_location("chamferdist.chamfer", os.path.join(CHAMFERDIST, "chamfer.py"))
    ch = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ch)
    pkg.ChamferDistance = ch.ChamferDistance
    return ch


def main():
    _install_chamferdist()
    spec = importlib.util.spec_from_file_location("ref_eval_utils", EVAL_UTILS)
    eu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(eu)
    import ref_shim
    e2e = ref_shim.load_functions("utils/e2e_predictor_utils.py",
                                  ("get_inside_mask", "compute_chamfer_distance", "compute_chamfer_distance_inner"))
    e2e["compute_chamfer_distance"].__globals__["chamfer_distance"] = sys.modules["chamferdist"].ChamferDistance()
    rec = {}
    for k, (pred, gt, origin) in enumerate(cases()):
        rec[f"pred_{k}"], rec[f"gt_{k}"], rec[f"origin_{k}"] = pred, gt, origin
        cd = e2e["compute_chamfer_distance_inner"](torch.from_numpy(pred), torch.from_numpy(gt), PC_RANGE)
        rec[f"chamfer_{k}"] = np.float64(float(cd))
        l1, absrel = eu.compute_ray_errors(pred, gt, origin, "cpu")
        rec[f"l1_{k}"], rec[f"absrel_{k}"] = np.float64(l1), np.float64(absrel)
        # intermediates, by the same statements of compute_ray_errors (eval_utils.py:186-215)
        th_h, ph_h, d_h = eu.spherical_projection(pred - origin[None, :])
        th, ph, d = eu.spherical_projection(gt - origin[None, :])
        mh, m = d_h > 1e-2, d > 1e-2
        ps = np.stack([th_h[mh], ph_h[mh], np.ones_like(th_h[mh])], axis=1)
        gs = np.stack([th[m], ph[m], np.ones_like(th[m])], axis=1)
        _, info = eu.chamfer_distance(torch.from_numpy(ps[None]), torch.from_numpy(gs[None]), reverse=True,
                                      reduction="mean")
        interp = eu.compute_ray_errors(pred, gt, origin, "cpu", return_interpolated_pcd=True)
        go, gc, inv = eu.clamp(gt[m], origin, return_invalid_mask=True)
        _, ic, _ = eu.clamp(interp, origin, return_invalid_mask=True)
        rec.update({f"theta_hat_{k}": th_h, f"phi_hat_{k}": ph_h, f"theta_{k}": th, f"phi_{k}": ph,
                    f"pred_idx_{k}": info[1].numpy()[0], f"interp_{k}": interp, f"clamped_gt_{k}": gc,
                    f"clamped_origin_{k}": go, f"clamped_interp_{k}": ic, f"invalid_{k}": inv})
        print(k, len(pred), len(gt), float(cd), float(l1), float(absrel), int(inv.sum()))
    rec["n_frames"] = np.int64(len(cases()))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "eval.npz"), **rec)


if __name__ == "__main__":
    main()
