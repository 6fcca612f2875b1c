"""ViDAR's evaluation metrics on the host: the oracle against goldens made by the reference's own eval_utils.py,
argument validation of the new C entry points, and summarize() against the dataset's arithmetic."""
import ctypes
import os

import numpy as np
import pytest

from oracle import eval_ref
from tests.eval_cases import PC_RANGE

GOLD = os.path.join(os.path.dirname(__file__), "golden", "eval.npz")


def golden_frames():
    g = np.load(GOLD)
    return g, [(g[f"pred_{k}"], g[f"gt_{k}"], g[f"origin_{k}"]) for k in range(int(g["n_frames"]))]


def spherical_mismatches(g, k, pred, gt, origin, idx):
    """Kept gt points whose NN index `idx` differs from the reference's.  Each must be explained by the one
    statement evaluated differently on purpose: the reference's float32 arctan2 and the fp64-rounded one differ
    on the gt point or on either pred point involved, or the best two spherical distances (fp32, fp64-rounded
    angles) are within 2 ulp.  Returns the mismatch mask over the kept gt points."""
    th_h, ph_h, d_h = eval_ref.spherical_projection(pred - origin[None])
    th, ph, d = eval_ref.spherical_projection(gt - origin[None])
    mh, m = d_h > np.float32(1e-2), d > np.float32(1e-2)
    ref_idx = g[f"pred_idx_{k}"]
    bad = idx != ref_idx
    if not bad.any():
        return bad
    gdiff = ((th != g[f"theta_{k}"]) | (ph != g[f"phi_{k}"]))[m]
    pdiff = ((th_h != g[f"theta_hat_{k}"]) | (ph_h != g[f"phi_hat_{k}"]))[mh]
    ps = np.stack([th_h[mh], ph_h[mh]], 1)
    gs = np.stack([th[m], ph[m]], 1)[bad]
    dd = (gs[:, None, 0] - ps[None, :, 0]) ** 2 + (gs[:, None, 1] - ps[None, :, 1]) ** 2
    two = np.sort(dd, axis=1)[:, :2]
    close = two[:, 1] - two[:, 0] <= 2 * np.spacing(two[:, 0])
    explained = gdiff[bad] | pdiff[idx[bad]] | pdiff[ref_idx[bad]] | close
    assert explained.all(), f"frame {k}: unexplained NN differences at {np.nonzero(bad)[0][~explained][:10]}"
    return bad


def test_oracle_matches_reference_goldens():
    g, frames = golden_frames()
    total, differ = 0, 0
    for k, (pred, gt, origin) in enumerate(frames):
        (l1, absrel), it = eval_ref.compute_ray_errors(pred, gt, origin, return_intermediates=True)
        np.testing.assert_allclose([l1, absrel], [g[f"l1_{k}"], g[f"absrel_{k}"]], rtol=1e-5, err_msg=f"frame {k}")
        np.testing.assert_allclose(eval_ref.compute_chamfer_distance_inner(pred, gt, PC_RANGE), g[f"chamfer_{k}"],
                                   rtol=1e-5, err_msg=f"frame {k}")
        # clamping the gt points does not depend on the search: bit-identical everywhere
        np.testing.assert_array_equal(it["clamped_gt"], g[f"clamped_gt_{k}"])
        np.testing.assert_array_equal(it["invalid"], g[f"invalid_{k}"])
        bad = spherical_mismatches(g, k, pred, gt, origin, it["idx"])
        np.testing.assert_array_equal(it["interp"][~bad], g[f"interp_{k}"][~bad])
        np.testing.assert_array_equal(it["clamped_interp"][~bad], g[f"clamped_interp_{k}"][~bad])
        total += len(bad)
        differ += int(bad.sum())
    print(f"NN differences explained by arctan2 rounding or near ties: {differ} of {total} kept gt points")
    assert differ < 1e-3 * total


def test_oracle_branches_are_exercised():
    """The cases reach every branch they are meant to: invalid (missed) rays, the 0.0 Chamfer value,
    points beyond the volume, and points within 1e-2 of the origin."""
    g, frames = golden_frames()
    assert g["invalid_4"].sum() > 0
    assert float(g["chamfer_6"]) == 0.0
    assert any((np.abs(gt) > 70).any() for _, gt, _ in frames)
    assert any((np.linalg.norm(gt - o, axis=1) <= 1e-2).any() for _, gt, o in frames)


def test_oracle_failure_types():
    o = np.zeros(3, np.float32)
    gt = np.array([[5.0, 1.0, 0.5]], np.float32)
    with pytest.raises(ValueError):
        eval_ref.compute_ray_errors(np.zeros((2, 3), np.float32), gt, o)
    # the interpolated point rounds back onto a far origin: a degenerate ray
    o2 = np.array([1e6, 0.0, 0.0], np.float32)
    with pytest.raises(RuntimeError):
        eval_ref.compute_ray_errors(np.array([[1e6, 0.02, 0.0]], np.float32),
                                    np.array([[1e6 + 0.0625, 0.0, 0.0]], np.float32), o2)
    # a pred point at infinity interpolates to (inf, nan, nan), which no plane brings back
    with pytest.raises(AssertionError):
        eval_ref.compute_ray_errors(np.array([[np.inf, 3.0, 0.0]], np.float32), gt, o)
    assert np.isnan(eval_ref.compute_ray_errors(np.zeros((3, 3), np.float32), np.zeros((2, 3), np.float32), o)[0])


def test_summarize_matches_dataset_evaluate():
    from vidar_b200.evaluate import summarize
    rng = np.random.default_rng(0)
    results = [{f"frame.{f}": dict(count=2, chamfer_distance=float(rng.random()), l1_error=float(rng.random()),
                                   absrel_error=float(rng.random())) for f in range(3)} for _ in range(4)]
    want = {}
    for f in range(3):
        k = f"frame.{f}"
        c = sum(r[k]["count"] for r in results)
        want[k] = dict(count=c, **{m: sum(r[k][m] for r in results) / c
                                   for m in ("chamfer_distance", "l1_error", "absrel_error")})
    got = summarize(results)
    assert got.keys() == want.keys()
    for k in want:
        assert got[k]["count"] == want[k]["count"]
        for m in ("chamfer_distance", "l1_error", "absrel_error"):
            assert got[k][m] == pytest.approx(want[k][m], rel=1e-15)
    assert results[0]["frame.0"]["count"] == 2          # inputs untouched
    assert summarize([]) == {}


def test_argument_validation_of_the_eval_entry_points():
    """Runs on a thread of its own: the last-error text is per thread, and other tests expect it empty."""
    import threading
    err = []

    def run():
        try:
            _validate_eval_entry_points()
        except BaseException as e:      # re-raised on the test's thread
            err.append(e)
    t = threading.Thread(target=run)
    t.start()
    t.join()
    if err:
        raise err[0]


def _validate_eval_entry_points():
    from vidar_b200 import _lib
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    cases = [
        (L.vidar_nn_segments_forward, (X, X, N, X, X, X, X, X, X, 3, 10, 5, 5, N), b"null pointer"),
        (L.vidar_nn_segments_forward, (X, X, X, X, X, X, X, X, X, 0, 10, 5, 5, N), b"bad sizes"),
        (L.vidar_nn_segments_forward, (X, X, X, X, X, X, X, X, X, 3, -1, 5, 5, N), b"bad sizes"),
        (L.vidar_nn_segments_forward, (N, X, X, X, X, X, X, X, X, 3, 10, 5, 5, N), b"null query"),
        (L.vidar_nn_segments_forward, (X, N, X, X, X, X, X, X, X, 3, 10, 5, 5, N), b"null candidate"),
        (L.vidar_eval_prologue, (X, X, X, X, X, N, X, X, X, X, X, X, 2, 10, 10, N), b"null pointer"),
        (L.vidar_eval_prologue, (X, X, X, X, X, X, X, X, X, X, X, X, 0, 10, 10, N), b"bad sizes"),
        (L.vidar_eval_prologue, (X, X, X, X, X, X, X, X, X, X, X, X, 30000, 10, 10, N), b"bad sizes"),
        (L.vidar_eval_prologue, (N, X, X, X, X, X, X, X, X, X, X, X, 2, 10, 10, N), b"null point buffer"),
        (L.vidar_eval_prologue, (X, X, X, X, X, X, N, X, X, X, X, X, 2, 10, 10, N), b"null output buffer"),
        (L.vidar_eval_metrics, (X, X, X, X, X, X, X, X, X, X, N, X, 2, 10, N), b"null pointer"),
        (L.vidar_eval_metrics, (X, X, X, X, X, X, X, X, X, X, X, X, 0, 10, N), b"bad sizes"),
        (L.vidar_eval_metrics, (X, X, X, X, X, X, X, N, X, X, X, X, 2, 10, N), b"null point / search buffer"),
    ]
    for fn, args, needle in cases:
        rc = fn(*args)
        assert rc == 1, (fn.__name__, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (fn.__name__, L.vidar_last_error())
    # an empty query set is a valid no-op that launches nothing
    n0 = _lib.launch_count()
    assert L.vidar_nn_segments_forward(N, N, X, X, N, N, N, N, N, 3, 0, 0, 0, N) == 0
    assert _lib.launch_count() == n0
