"""The BEV encoder's front end on the GPU at training size: `point_sampling` (csrc/sca_glue.cu), the
camera projection every SpatialCrossAttention layer uses, and `compact_visible`'s per-camera pillar
lists and 1 / #cameras normaliser, against oracle/encoder_front_ref.py.

point_sampling's arithmetic is pinned (`__fmul_rn` / `__fadd_rn` / `__fdiv_rn` and one fmaf chain per
coordinate), so its coordinates and mask must equal the fp32 emulation bit for bit, on every element,
masked or not.  Against fp64 the mask may differ only on the ambiguity set (points whose margin to the
z = eps plane or to an image border is within twice its rounding bound), which must stay below 1e-4 of
the points, and coordinates in front of the camera must be within twice their bound.  The reference's
own fp32 statements (repeat + matmul with TF32 off + masks) must decide like the kernel outside the
ambiguity set.  Sizes, ratios and agreement fractions are printed (pytest -s).
"""
import numpy as np
import pytest
import torch

from oracle import encoder_front_ref as efr
from tests import geometry_cases as gc
from vidar_b200 import bev_geometry as geo
from vidar_b200 import sca

pytestmark = pytest.mark.gpu
SAFETY = 2.0


def _metas(l2i, img_hw):
    return [dict(lidar2img=m, img_shape=[tuple(img_hw) + (3,)] * len(m)) for m in l2i]


def _run(ref, l2i, pc_range, img_hw, cuda):
    cam, mask = geo.point_sampling(torch.from_numpy(ref).to(cuda), pc_range, _metas(l2i, img_hw))
    return cam.cpu().numpy(), mask.cpu().numpy()


def _reference_statements(ref, l2i, pc_range, img_hw, cuda):
    """encoder.py:94-156 restated: [D, B, cams, Q, 4, 4] repeat, fp32 matmul without TF32, eps masks."""
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        r = torch.from_numpy(ref).to(cuda).clone()
        for i in range(3):
            r[..., i:i + 1] = r[..., i:i + 1] * (pc_range[i + 3] - pc_range[i]) + pc_range[i]
        r = torch.cat((r, torch.ones_like(r[..., :1])), -1).permute(1, 0, 2, 3)
        D, B, Q = r.shape[:3]
        m = torch.from_numpy(np.asarray(l2i, np.float32)).to(cuda)
        cams = m.shape[1]
        r = r.view(D, B, 1, Q, 4).repeat(1, 1, cams, 1, 1).unsqueeze(-1)
        m = m.view(1, B, cams, 1, 4, 4).repeat(D, 1, 1, Q, 1, 1)
        p = torch.matmul(m, r).squeeze(-1)
        eps = 1e-5
        mask = p[..., 2:3] > eps
        uv = p[..., 0:2] / torch.maximum(p[..., 2:3], torch.ones_like(p[..., 2:3]) * eps)
        uv[..., 0] /= img_hw[1]
        uv[..., 1] /= img_hw[0]
        mask = mask & (uv[..., 1:2] > 0.0) & (uv[..., 1:2] < 1.0) & (uv[..., 0:1] < 1.0) & (uv[..., 0:1] > 0.0)
        return uv.permute(2, 1, 3, 0, 4).cpu().numpy(), mask.permute(2, 1, 3, 0, 4).squeeze(-1).cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32


def _check_lists(mask, cuda):
    idx, count, inv = sca.compact_visible(torch.from_numpy(np.ascontiguousarray(mask)).to(cuda))
    want_idx, want_count, want_inv = efr.visible_lists(mask)
    count, idx = count.cpu().numpy(), idx.cpu().numpy()
    assert np.array_equal(count, want_count)
    for c, w in enumerate(want_idx):
        assert np.array_equal(idx[c, :len(w)], w), f"camera {c}"
    assert np.array_equal(inv.cpu().numpy().view(np.uint32), want_inv.view(np.uint32))
    return want_inv


@pytest.mark.parametrize("img_hw", [(928, 1600), (900, 1600)])
@pytest.mark.parametrize("bs", [1, 2])
def test_point_sampling_at_training_size(cuda, bs, img_hw):
    ref = geo.get_reference_points(200, 200, 8, 4, "3d", bs, "cpu").numpy()
    l2i = np.stack([m["lidar2img"] for m in gc.rig(2)])[:bs]       # sample 1's rig differs from sample 0's
    cam, mask = _run(ref, l2i, gc.PC_RANGE, img_hw, cuda)
    # (a) bit-identical to the emulation of the kernel's statements
    ecam, emask = efr.point_sampling_fp32(ref, l2i, gc.PC_RANGE, img_hw)
    assert cam.shape == ecam.shape == (6, bs, 40000, 4, 2)
    assert np.array_equal(mask, emask)
    assert np.array_equal(cam.view(np.uint32), ecam.view(np.uint32))
    # (b) the fp64 mask outside the ambiguity set
    o = efr.point_sampling_fp64(ref, l2i, gc.PC_RANGE, img_hw)
    amb = efr.ambiguous(o, SAFETY)
    assert not (mask != o["mask"])[~amb].any()
    assert amb.mean() < 1e-4
    # (c) coordinates one metre or more in front of the camera within their bound of fp64
    front = o["pz_eps"] > 1.0
    ratios = [float((np.abs(cam[..., i] - o["ref_cam"][..., i])[front] / (SAFETY * o[k][front])).max())
              for i, k in ((0, "u_bound"), (1, "v_bound"))]
    assert max(ratios) < 1
    # (d) the reference's own statements on the GPU
    rcam, rmask = _reference_statements(ref, l2i, gc.PC_RANGE, img_hw, cuda)
    assert not (rmask != mask)[~amb].any()
    same = (rcam.view(np.uint32) == cam.view(np.uint32)).all(-1)
    print(f"\nbs={bs} {img_hw}: ambiguity set {amb.sum()} / {amb.size}, kernel != fp64 mask on {(mask != o['mask']).sum()},"
          f" reference statements != kernel mask on {(rmask != mask).sum()}; coordinate error / bound u {ratios[0]:.3e}"
          f" v {ratios[1]:.3e}; reference coordinates bit-identical to the kernel's: {same.mean():.4f}")
    # visible lists on masks from the rig: adjacent cameras overlap, so some pillars are seen twice
    inv = _check_lists(mask, cuda)
    assert (inv == np.float32(0.5)).any()
    if bs == 2:
        assert not np.array_equal(mask[:, 0], mask[:, 1])
        assert not np.array_equal(inv[0], inv[1])


@pytest.mark.parametrize("D", [1, 8])
def test_point_sampling_non_square_bev(cuda, D):
    """50 x 120 BEV: a swap of the Q / D / sample / camera indexing or of the two axes shows."""
    ref = geo.get_reference_points(50, 120, 8, D, "3d", 2, "cpu").numpy()
    l2i = np.stack([m["lidar2img"] for m in gc.rig(2)])
    cam, mask = _run(ref, l2i, gc.PC_RANGE, (928, 1600), cuda)
    ecam, emask = efr.point_sampling_fp32(ref, l2i, gc.PC_RANGE, (928, 1600))
    assert np.array_equal(mask, emask) and np.array_equal(cam.view(np.uint32), ecam.view(np.uint32))
    assert mask.any() and not mask.all()
    _check_lists(mask, cuda)


def _edge_case():
    """Rows built so every projection is exact: pc_range [0, 1]^3 makes (x, y, z) = ref, and camera c
    maps p = (W s_c x, H s_c y, s_c) with s_c its depth, so u = x and v = y up to the divisions'
    rounding.  Points land on u, v in {0, 1} (excluded by the strict inequalities), just inside them, at
    p.z == 1e-5f (excluded), one fp32 step above it (kept), and behind the camera (divided by eps)."""
    H, W = 928.0, 1600.0
    eps = np.float32(1e-5)
    depths = [np.float32(1), eps, np.nextafter(eps, np.float32(1)), np.float32(-1), np.float32(37.5)]
    l2i = np.zeros((1, len(depths), 4, 4), np.float32)
    for c, s in enumerate(depths):
        l2i[0, c, 0, 0], l2i[0, c, 1, 1], l2i[0, c, 2, 3], l2i[0, c, 3, 3] = W * s, H * s, s, 1
    vals = np.array([0, 2.0 ** -24, 0.25, 0.5, 1 - 2.0 ** -24, 1], np.float32)
    xs, ys = np.meshgrid(vals, vals, indexing="ij")
    ref = np.stack((xs.ravel(), ys.ravel(), np.full(xs.size, 0.5, np.float32)), -1)[None, None]   # [1,1,36,3]
    return ref, l2i, [0.0, 0.0, 0.0, 1.0, 1.0, 1.0], (928, 1600), vals


def test_point_sampling_exact_edges(cuda):
    ref, l2i, pc, img_hw, vals = _edge_case()
    cam, mask = _run(ref, l2i, pc, img_hw, cuda)
    ecam, emask = efr.point_sampling_fp32(ref, l2i, pc, img_hw)
    assert np.array_equal(mask, emask) and np.array_equal(cam.view(np.uint32), ecam.view(np.uint32))
    x, y = ref[0, 0, :, 0], ref[0, 0, :, 1]
    inside = (x > 0) & (x < 1) & (y > 0) & (y < 1)
    for c in (0, 2, 4):                                   # in front: kept exactly when strictly inside
        assert np.array_equal(mask[c, 0, :, 0], inside), f"camera {c}"
    assert not mask[1].any()                              # p.z == eps
    assert not mask[3].any()                              # behind the camera
    # on the borders the coordinate itself is exact
    on = (x == 0) | (x == 1) | (y == 0) | (y == 1)
    assert np.array_equal(cam[0, 0, :, 0, 0][x == 0], x[x == 0]) and np.array_equal(cam[0, 0, :, 0, 0][x == 1], x[x == 1])
    assert np.array_equal(cam[0, 0, :, 0, 1][y == 0], y[y == 0]) and np.array_equal(cam[0, 0, :, 0, 1][y == 1], y[y == 1])
    assert on.sum() == 20
    # behind the camera: p.xy / eps / (W, H) = -(x, y) / eps
    np.testing.assert_allclose(cam[3, 0, :, 0], -np.stack((x, y), -1) / np.float64(np.float32(1e-5)), rtol=1e-6)


@pytest.mark.parametrize("D", [1, 4, 8])
@pytest.mark.parametrize("Q", [1, 31, 32, 1023, 1024, 1025, 2048, 40000])
def test_compact_visible_block_scan_edges(cuda, Q, D):
    """One camera per pattern: random, every pillar, none, only pillar 0, only pillar Q - 1, visible only
    through d = D - 1, exactly the first min(Q, 1024) pillars (a list ending on a 1024-pillar chunk);
    batch element 1 differs from element 0 everywhere the pattern is random."""
    rng = np.random.default_rng(Q * 10 + D)
    m = np.zeros((7, 2, Q, D), bool)
    m[0] = rng.random((2, Q, D)) < 0.1
    m[1] = True
    m[3, :, 0, rng.integers(D)] = True
    m[4, :, Q - 1, rng.integers(D)] = True
    m[5, :, :, D - 1] = rng.random((2, Q)) < 0.5
    m[6, :, :1024] = True
    m[6, 1] = rng.random((Q, D)) < 0.3
    _check_lists(m, cuda)
