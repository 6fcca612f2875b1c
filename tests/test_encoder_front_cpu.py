"""Host checks of oracle/encoder_front_ref.py, the oracle the encoder front-end and projection GPU tests
judge the kernels by, and of point_sampling's input validation.

* `fmaf` is the exact rounding of a * b + c (against `fractions.Fraction`), midpoint cases included.
* On the full 200 x 200 BEV, 4 anchors, 6 cameras, 2 samples with different rigs, the fp32 emulation of the
  kernel decides every point as fp64 does outside the ambiguity set, and its coordinates are within
  their bound: the GPU tests' criteria are not tighter than fp32 allows.
* Every projection bound holds for fp32 computations in another order (torch F.linear, row sums in
  chunks), and is exceeded by a computation that drops one row tile or one product term: the bounds
  are neither vacuous nor tighter than fp32 allows.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import encoder_front_ref as efr
from tests import geometry_cases as gc
from tests import latent_cases as lc
from vidar_b200 import bev_geometry as geo

SAFETY = 2.0


def test_fmaf_is_correctly_rounded():
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(np.float32)
    # midpoints: c = 2^k (2^24 + 2j) lies on the fp32 grid of spacing 2^(k+1), and a b = 2^k (1 -+ 2^-46)
    # puts the exact sum 2^-46 relative below / above the midpoint 2^k (2^24 + 2j + 1), where fp64
    # rounds it onto the midpoint: a plain fp32(fp64 sum) then rounds a second time, to even.
    k = rng.integers(-20, 20, 400)
    j = rng.integers(0, 1 << 22, 400)
    sgn = rng.choice([-1.0, 1.0], 400)
    one_p = np.float32(1 + 2.0 ** -23)
    cm = (sgn * np.ldexp(2.0 ** 24 + 2 * j, k)).astype(np.float32)
    am = (sgn * np.ldexp(one_p, k)).astype(np.float32)
    bm = np.where(rng.random(400) < 0.5, np.float32(1 - 2.0 ** -23), one_p).astype(np.float32)
    a, b, c = np.concatenate((a, am)), np.concatenate((b, bm)), np.concatenate((c, cm))
    got = efr.fmaf(a, b, c)
    want = np.array([efr.fraction_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    assert (naive[n:] != want[n:]).sum() > 50                 # the midpoint cases do defeat double rounding


def _front_case():
    ref = geo.get_reference_points(200, 200, 8, 4, "3d", 2, "cpu").numpy()
    metas = gc.rig(2)
    l2i = np.stack([m["lidar2img"] for m in metas])
    return ref, l2i


def test_emulation_decides_like_fp64_outside_the_ambiguity_set():
    ref, l2i = _front_case()
    cam, mask = efr.point_sampling_fp32(ref, l2i, gc.PC_RANGE, gc.IMG_SHAPE[:2])
    o = efr.point_sampling_fp64(ref, l2i, gc.PC_RANGE, gc.IMG_SHAPE[:2])
    amb = efr.ambiguous(o, SAFETY)
    assert mask.shape == (6, 2, 40000, 4) and cam.shape == (6, 2, 40000, 4, 2)
    assert not (mask != o["mask"])[~amb].any()
    print(f"\nambiguity set: {amb.sum()} of {amb.size} points; emulation differs from fp64 on {(mask != o['mask']).sum()}")
    assert amb.mean() < 1e-4
    assert 0.05 < mask.mean() < 0.5 and mask[:, 0].any() and mask[:, 1].any()
    front = o["pz_eps"] > 1.0                                 # one metre in front of the camera
    for i, key in ((0, "u_bound"), (1, "v_bound")):
        err = np.abs(cam[..., i].astype(np.float64) - o["ref_cam"][..., i])[front]
        ratio = (err / (SAFETY * o[key][front])).max()
        print(f"coordinate {'uv'[i]}: largest error / bound {ratio:.3e}")
        assert ratio < 1


def _chunked_rows(a, b, chunk=1000):
    """a^T b summed over rows chunk by chunk in fp32: a row order unlike the kernels'."""
    acc = torch.zeros(a.shape[1], b.shape[1])
    for r in range(0, a.shape[0], chunk):
        acc += a[r:r + chunk].t() @ b[r:r + chunk]
    return acc


@pytest.mark.parametrize("rows,E,D", [(40000, 256, 16), (16897, 128, 8), (9000, 256, 4)])
def test_projection_bounds_hold_for_fp32_in_another_order(rows, E, D):
    t = lc.proj_inputs(rows, E, D, seed=rows)
    d = {k: v.double() for k, v in t.items()}
    ref = efr.proj_reference(**d)
    per = E // D
    # fp32 CPU computation, every sum in an order the kernels do not use
    qe = t["prob"].repeat_interleave(per, -1)
    lin = F.linear(t["pooled"], t["w_b"], t["b_b"])
    gl = t["g_out"] * qe
    g = torch.Generator().manual_seed(1)
    acc = {"grad_w_occ": torch.randn(D, E, generator=g), "grad_w_b": torch.randn(E, 16, generator=g),
           "grad_b_b": torch.randn(E, generator=g)}
    got = dict(occ=F.linear(t["x"], t["w_occ"], t["b_occ"]), feat=F.linear(t["x"], t["w_feat"], t["b_feat"]),
               out=lin * qe, grad_embed=t["g_occ"] @ t["w_occ"] + t["g_feat"] @ t["w_feat"],
               grad_w_occ=acc["grad_w_occ"] + _chunked_rows(t["g_occ"], t["x"]),
               grad_b_occ=_chunked_rows(t["g_occ"], torch.ones(rows, 1))[:, 0],
               grad_w_feat=_chunked_rows(t["g_feat"], t["x"], 4096), grad_b_feat=t["g_feat"].sum(0),
               grad_pooled=gl @ t["w_b"], grad_prob=(t["g_out"] * lin).view(rows, D, per).sum(-1),
               grad_w_b=acc["grad_w_b"] + _chunked_rows(gl, t["pooled"]),
               grad_b_b=acc["grad_b_b"] + gl.sum(0))
    want = dict(ref)
    for k, a0 in acc.items():
        want[k] = ref[k] + a0.double()
    bounds = efr.proj_bounds(d, 132, {k: v.double() for k, v in acc.items()})
    for k, bnd in bounds.items():
        err = (got[k].double() - want[k]).abs()
        ratio = float((err / (SAFETY * bnd)).max())
        print(f"\n{k:12s} rows={rows} E={E} D={D}: largest fp32 error / bound {ratio:.3e}")
        assert ratio < 1, k
    # not vacuous: one 32-row tile left out of a weight gradient, one product term left out of an output
    miss = (got["grad_w_occ"] - t["g_occ"][64:96].t() @ t["x"][64:96]).double() - want["grad_w_occ"]
    assert float((miss.abs() / (SAFETY * bounds["grad_w_occ"])).max()) > 1
    short = F.linear(t["x"][:, 1:], t["w_occ"][:, 1:], t["b_occ"]).double() - want["occ"]
    assert float((short.abs() / (SAFETY * bounds["occ"])).max()) > 1


def test_proj_launch_geometry():
    # rows of one round on a 132-SM card: 264 blocks x 32 (backward), 264 x 64 and 528 x 32 (forward)
    assert efr.proj_launch("proj_in_bwd", 40000, 132) == (264, 8448, 160)
    assert efr.proj_launch("proj_out_bwd", 40000, 132) == (264, 8448, 160)
    assert efr.proj_launch("proj_in_fwd", 40000, 132) == (264, 16896, 192)
    assert efr.proj_launch("proj_out_fwd", 40000, 132) == (528, 16896, 96)
    assert efr.proj_launch("proj_in_bwd", 1, 132) == (1, 32, 32)


def test_visible_lists():
    mask = np.zeros((3, 2, 5, 2), bool)
    mask[0, 0, 1, 1] = mask[0, 0, 4, 0] = True
    mask[1, 0, 4, 1] = mask[1, 1, 2, 0] = True
    mask[2, 1, 0, 0] = True
    idx, counts, inv = efr.visible_lists(mask)
    assert [i.tolist() for i in idx] == [[1, 4], [4], []] and counts.tolist() == [2, 1, 0]
    assert inv.dtype == np.float32 and inv.tolist() == [[1, 1, 1, 1, 0.5], [1, 1, 1, 1, 1]]


def test_point_sampling_validates_inputs_before_launch():
    ref = geo.get_reference_points(4, 5, 8, 2, "3d", 2, "cpu")
    metas = gc.rig(2)
    with pytest.raises(RuntimeError, match="1 img_metas for 2 samples"):
        geo.point_sampling(ref, gc.PC_RANGE, metas[:1])
    bad = [dict(metas[0]), dict(metas[1])]
    bad[1]["lidar2img"] = metas[1]["lidar2img"][:, :3]
    with pytest.raises(RuntimeError, match=r"lidar2img of sample 1 must be \[num_cams, 4, 4\]"):
        geo.point_sampling(ref, gc.PC_RANGE, bad)
    bad[1]["lidar2img"] = metas[1]["lidar2img"][0]
    with pytest.raises(RuntimeError, match=r"must be \[num_cams, 4, 4\]"):
        geo.point_sampling(ref, gc.PC_RANGE, bad)
    bad[1]["lidar2img"] = metas[1]["lidar2img"][:5]
    with pytest.raises(RuntimeError, match="sample 1 has 5 cameras, sample 0 has 6"):
        geo.point_sampling(ref, gc.PC_RANGE, bad)
    for rng in (gc.PC_RANGE[:5], gc.PC_RANGE + [1.0], [float("nan")] + gc.PC_RANGE[1:], [float("inf")] * 6):
        with pytest.raises(RuntimeError, match="pc_range must be 6 finite numbers"):
            geo.point_sampling(ref, rng, metas)
    with pytest.raises(RuntimeError, match=r"reference_points must be \[bs, D, num_query, 3\]"):
        geo.point_sampling(ref[0], gc.PC_RANGE, metas)
    # valid inputs get as far as the device check
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        geo.point_sampling(ref, gc.PC_RANGE, metas)
