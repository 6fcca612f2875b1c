"""Pin the CPU oracle (oracle/dvr_ref.c) against outputs of the REFERENCE's own CUDA kernels
(third_lib/dvr, third_lib/dvxlr, dvxlr_v2 compiled unmodified-in-arithmetic by
oracle/build_ref.py and run on the GPU; vectors made by tools/make_golden_dvr.py)."""
import glob
import os

import numpy as np
import pytest

from oracle import dvr_ref

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "dvr_*.npz")))


def _close(a, b, what, rtol=1e-5, atol_scale=1e-6):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = np.sqrt((b ** 2).mean()) + 1e-30
    err = np.abs(a - b)
    tol = rtol * np.abs(b) + atol_scale * scale
    assert (err <= tol).all(), f"{what}: max err {err.max():.3e} (scale {scale:.3e}), {(err > tol).sum()} bad"


@pytest.mark.skipif(not GOLD, reason="golden vectors not generated yet (tools/make_golden_dvr.py on a GPU box)")
@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_oracle_reproduces_reference_cuda_outputs(path):
    g = np.load(path)
    s, o, p, t, r = g["sigma"], g["origin"], g["points"], g["tindex"], g["sigma_regul"]
    np.testing.assert_array_equal(dvr_ref.init(p, t, list(s.shape[1:])), g["occupancy"])
    for ph in ("test", "train"):
        pred, gt = dvr_ref.render_forward(s, o, p, t, None, ph)
        _close(pred, g[f"fwd_{ph}_pred"], f"render_forward {ph} pred")
        _close(gt, g[f"fwd_{ph}_gt"], f"render_forward {ph} gt")
    for loss in ("l1", "l2", "absrel"):
        pred, gt, grad = dvr_ref.render(s, o, p, t, loss)
        _close(pred, g[f"render_{loss}_pred"], f"render {loss} pred")
        _close(gt, g[f"render_{loss}_gt"], f"render {loss} gt")
        # the reference's gradient is a racy `+=` (dvr.cu:621-622): lost updates only ever
        # drop terms, so it can differ; require agreement on the bulk of the volume
        ref = g[f"render_{loss}_grad_racy"]
        scale = np.abs(grad).max()
        frac_close = (np.abs(grad - ref) <= 1e-4 * scale).mean()
        assert frac_close > 0.90, f"render {loss}: only {frac_close:.3f} of grad_sigma agrees with the racy reference"
    k = int(g["dvxlr_k"])
    pred, gt, dd, idx, ray_pred, ind = dvr_ref.dvxlr_render(s, o, p, t, r)
    _close(pred, g["dvxlr_pred"], "dvxlr pred")
    _close(gt, g["dvxlr_gt"], "dvxlr gt")
    count = (ind >= 0).sum(-1)
    np.testing.assert_array_equal(count, g["dvxlr_count"])
    assert count.max() == k
    np.testing.assert_array_equal(idx[:, :, :k].astype(np.int16), g["dvxlr_idx"])
    np.testing.assert_array_equal(ind[:, :, :k].astype(np.int8), g["dvxlr_indicator"])
    np.testing.assert_array_equal(ray_pred[:, :, :k], g["dvxlr_ray_pred"])
    _close(dd[:, :, :k], g["dvxlr_dd"], "dd_dsigma", rtol=1e-4)
    assert not dd[:, :, k:].any() and not idx[:, :, k:].any()
    rng = np.random.default_rng(123)
    rng.standard_normal(s.shape)                       # same stream as the generator script
    gp = rng.standard_normal(pred.shape).astype(np.float32)
    grp = rng.standard_normal(ray_pred.shape).astype(np.float32)
    np.testing.assert_array_equal(gp, g["grad_pred"])
    em = gp[..., None] * dd
    ga, gb = dvr_ref.dvxlr_get_grad_sigma(em, idx, t, s, ind, grp)
    _close(ga, g["scatter_grad_sigma"], "get_grad_sigma_v2 grad_sigma", rtol=1e-4, atol_scale=1e-5)
    _close(gb, g["scatter_grad_regul"], "get_grad_sigma_v2 grad_sigma_regul", rtol=1e-4, atol_scale=1e-5)
    _close(ga, g["scatter_grad_sigma_v1"], "get_grad_sigma grad_sigma", rtol=1e-4, atol_scale=1e-5)
