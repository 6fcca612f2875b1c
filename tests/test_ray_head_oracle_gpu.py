"""Every entry point of vidar_b200/csrc/ray_head.cu against the fp64 oracle of oracle/ray_head_ref.py.

Each case compares every ray.  The inputs cross every lane boundary of the one-warp-per-ray mapping
(num_way + with_gt = 1 .. 1001 samples, lanes with no sample, lanes with up to 32), the block tail (R = 0, 1, 7,
8, 9), non-cubic grids with distinct sizes (an axis swap changes the result), Z = 1 and Y = 1, frames -1 and F
(skipped rows), `frame = None`, axis-aligned rays of both signs from an origin on the voxel lattice (waypoints on
integer and half-integer coordinates: weights of exactly 0 and 1, zero-weight corners outside the volume), GT
points exactly on the faces 0 and X / Y / Z and one fp32 step inside, origins outside the volume (waypoints that
enter late or never), and sigma with blocks of exact zeros, a constant 10 (exact ties) and +-60 (the online
log-sum-exp far from 0).

Tolerances, u = 2^-24 (oracle U32), A_k = sum_j |sigma_j w_j| of sample k (oracle absw):
- geometry: the kernels and the oracle run the same fp32 statements, so valid, the mask and the -inf pattern are
  equal, lengths within 1 ulp, and a decoded depth is bit-equal to the chosen waypoint's length.
- logit: each fp32 weight carries <= 5 roundings (two of its three factors may round, two products), the 8
  fused multiply-adds 8 more: |logit - fp64| <= C_LOGIT u A_k with C_LOGIT = 16.
- lse, ce, p_next: oracle.lse_cond (48 A for the logits, the running and the final max; per online step expf's
  2 ulp and the rounding of its argument, |v - m| <= 2 max|v|, over K/32 lane steps and 5 shuffle levels; log and
  the final add).  ce adds 16 A_0 and its own rounding; p_next = nx / S doubles the relative bound.
- arg-max: a logit + noise difference is off by at most u (32 max A + 2 |y| + 2) (oracle tie_cond); indices may
  differ only where the fp64 margin between best and second best is within that, and every such ray is reported.
  A margin of exactly 0 is an exact tie (lattice samples of the constant block): there the smallest index must win.
- ce_regularization_loss: the per-ray ce bounds weighted as the loss weights them, plus log2(rays) + 16
  roundings of the device sums.
- backward: per voxel, u (err + (count + 6) mag) (oracle.Scatter): the bound on each scattered dl_k, then 6
  roundings in w_j and dl_k w_j, and at most count - 1 roundings of a partial sum no larger than mag, whatever
  order the red.add reductions land in.
All bounds are first order; SAFETY = 2 covers the second-order terms.  The largest error-to-bound ratio of each
quantity is printed at the end of the module (pytest -s).
"""
import math

import numpy as np
import pytest
import torch

from oracle import ray_head_ref as ref
from vidar_b200 import _lib, ray_head

pytestmark = pytest.mark.gpu

U = ref.U32
C_LOGIT = 16
SAFETY = 2.0
TINY = 2.0 ** -125          # a product or reduction below fp32's smallest normal may flush: it loses less
RATIOS = {}
NEAR_TIES = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest error / bound per quantity:")
    for k in sorted(RATIOS):
        print(f"  {k:28s} {RATIOS[k]:.3e}")
    print(f"near-tie arg-max rays allowed to differ: {len(NEAR_TIES)}")
    for t in NEAR_TIES:
        print("  ", t)


def _within(what, err, bound):
    """err <= bound element-wise (err == 0 where bound == 0), recording the largest ratio."""
    err, bound = err.double().cpu().reshape(-1), bound.double().cpu().reshape(-1)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {err.numel()} outside the bound, worst err "
                           f"{err[bad].max():.3e} at bound {bound[bad][err[bad].argmax()]:.3e}")
    pos = bound > 0
    if pos.any():
        RATIOS[what] = max(RATIOS.get(what, 0.0), float((err[pos] / bound[pos]).max()))


def _scatter_ok(what, got, sc, extra=0):
    bound = SAFETY * U * (sc.err + (sc.count + 6 + extra) * sc.mag) + sc.count * TINY
    _within(what, (got.double().cpu() - sc.grad).abs(), bound)


def _ulp1(a, b):
    np.testing.assert_array_max_ulp(a.cpu().numpy(), b.cpu().numpy(), maxulp=1)


def _abi(name, dev, *args):
    """Call vidar_<name> on the current stream; tensors -> device pointers, None -> nullptr."""
    conv = [_lib.ptr(a) if (a is None or isinstance(a, torch.Tensor)) else a for a in args]
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), "vidar_" + name)(*conv, _lib.stream_ptr(dev)))
    torch.cuda.synchronize(dev)


# ---- inputs ----------------------------------------------------------------------------------------------------
def _n32(c, size):
    c, size = np.float32(c), np.float32(size)
    return np.float32(np.float32(c / size) * np.float32(2)) - np.float32(1)


def _first_true(pred, lo, hi):
    """Smallest fp32 c in [lo, hi] (non-negative, pred(hi) true, pred monotone) with pred(c), by bisection on
    the bit patterns, which order non-negative floats."""
    a, b = int(np.float32(lo).view(np.int32)), int(np.float32(hi).view(np.int32))
    while a < b:
        m = (a + b) // 2
        if pred(np.int32(m).view(np.float32)):
            b = m
        else:
            a = m + 1
    return np.int32(a).view(np.float32)


def _face_coords(size):
    """(0, first fp32 value inside, last fp32 value inside, size) along an axis of `size` voxels."""
    lo = _first_true(lambda c: _n32(c, size) > -1, 0.0, size)
    hi = np.nextafter(_first_true(lambda c: _n32(c, size) >= 1, 0.0, size), np.float32(0))
    assert _n32(np.nextafter(lo, np.float32(0)), size) <= -1 and _n32(hi, size) < 1
    return [0.0, float(lo), float(hi), float(size)]


def lattice_origin(grid):
    Z, Y, X = grid
    return torch.tensor([float(X // 2), Y // 2 + 0.5, Z // 2 + 0.5])


def make_case(grid, nf, seed, n_random=240):
    """sigma [nf,Z,Y,X], origin [nf,3], points [R,3], frame int32 [R] (with -1 and nf rows).
    Frame 0's origin lies on the voxel lattice (integer x, half-integer y, z) inside the volume; frame 1's just
    outside (-x side: waypoints enter late or never); frame 2's far outside (every waypoint masked)."""
    Z, Y, X = grid
    g = torch.Generator().manual_seed(seed)
    size = torch.tensor([X, Y, Z], dtype=torch.float32)
    o0 = lattice_origin(grid)
    origin = torch.stack([o0, torch.tensor([-6.3, 0.37 * Y + 0.1, 0.5 * Z + 0.05]),
                          torch.tensor([-3000.5, 0.5 * Y, 0.5 * Z])])[:nf].contiguous()
    sigma = torch.randn(nf, Z, Y, X, generator=g)
    ix, iy, iz = X // 2, Y // 2, Z // 2
    ys, zs = slice(max(iy - 1, 0), iy + 2), slice(max(iz - 1, 0), iz + 2)
    sigma[:, zs, ys, ix + 4:ix + 12] = 10.0                              # exact ties along +x from frame 0
    sigma[:, :, ys, max(ix - 2, 0):ix + 2] = 0.0                         # exact zeros: the column under o0
    big = sigma[:, :, :, max(ix - 12, 0):max(ix - 3, 0)]
    big.copy_(60 * torch.sign(torch.randn(big.shape, generator=g)) + torch.randn(big.shape, generator=g))
    pts, frames = [], []
    # random GT points, some outside, on every frame and on no frame
    pts.append(size * (1.3 * torch.rand(n_random, 3, generator=g) - 0.15))
    fr = torch.randint(0, nf, (n_random,), generator=g)
    u = torch.rand(n_random, generator=g)
    fr[u < 0.08] = -1
    fr[u > 0.95] = nf
    frames.append(fr)
    # axis-aligned rays of both signs from the lattice origin, ending inside and beyond the faces
    ax = []
    for a in range(3):
        for s in (-1.0, 1.0):
            for d in (0.75, 2.0, 5.0, 40.0, 2000.0):
                p = o0.clone()
                p[a] += s * d
                ax.append(p)
    plus_x = n_random + 5 + torch.arange(5)          # (a, s) = (0, +1): through the constant block
    pts.append(torch.stack(ax))
    frames.append(torch.zeros(len(ax), dtype=torch.long))
    # GT on the faces (invalid) and one fp32 step inside them (valid)
    fc = []
    for a in range(3):
        for c in _face_coords(int(size[a])):
            p = o0.clone()
            p[a] = c
            fc.append(p)
    pts.append(torch.stack(fc))
    frames.append(torch.zeros(len(fc), dtype=torch.long))
    if nf >= 3:         # GT inside, origin so far out that no waypoint is: the GT is the only unmasked sample
        pts.append(size * (0.1 + 0.8 * torch.rand(12, 3, generator=g)))
        frames.append(torch.full((12,), 2, dtype=torch.long))
    R = sum(p.shape[0] for p in pts)
    exact = torch.zeros(R, dtype=torch.bool)
    exact[plus_x] = all(v & (v - 1) == 0 for v in grid)                   # /size exact: lattice samples exact
    frame = torch.cat(frames).to(torch.int32).contiguous()
    return dict(sigma=sigma, origin=origin, points=torch.cat(pts).contiguous(), frame=frame, grid=grid, exact=exact,
                far=frame == 2)


def _exact_rows(c, step):
    """Rows whose tied maxima are exact in fp32 too (lattice samples of the constant block, step 1): there the
    smallest index must win; elsewhere an fp64 tie is an fp32 near tie."""
    return c["exact"] & (step == 1.0) if "exact" in c else torch.zeros(c["points"].shape[0], dtype=torch.bool)


CASES = {"5x13x29": ((5, 13, 29), 3), "lattice8x16x32": ((8, 16, 32), 3), "z1": ((1, 13, 29), 3),
         "y1": ((5, 1, 29), 1)}
COMBOS = ([("5x13x29", n) for n in (1, 31, 32, 33, 64, 512, 1000)]
          + [("lattice8x16x32", n) for n in (1, 31, 32, 33, 64, 512, 1000)]
          + [("z1", n) for n in (1, 33, 512)] + [("y1", n) for n in (1, 33, 512)])
STEP = {1: 1.0, 31: 1.0, 32: 0.5, 33: 1.0, 64: 0.5, 512: 0.125, 1000: 0.0625}     # lattice8x16x32: always 1
_cache = {}


def case(name):
    if name not in _cache:
        grid, nf = CASES[name]
        _cache[name] = make_case(grid, nf, seed=len(_cache) + 11)
    return _cache[name]


def _dev(c, cuda):
    return (c["sigma"].to(cuda), c["origin"].to(cuda), c["points"].to(cuda),
            None if c["frame"] is None else c["frame"].to(cuda))


def _dims(c):
    nf, Z, Y, X = c["sigma"].shape
    return c["points"].shape[0], nf, Z, Y, X


# ---- the checks, one per entry-point pair ---------------------------------------------------------------------
def check_sample(cuda, c, nw, step, tag):
    sigma, origin, points, frame = _dev(c, cuda)
    R = points.shape[0]
    for with_gt in (True, False):
        t = f"{tag} gt{int(with_gt)}"
        s = sigma.clone().requires_grad_(True)
        logits, length, valid = ray_head.ray_sample(s, origin, points, frame, nw, step, with_gt)
        lg64, ln64, vd64, absw = ref.sample_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, with_gt)
        assert torch.equal(valid.cpu() > 0, vd64), t
        assert torch.equal(logits.detach().cpu() == float("-inf"), lg64 == float("-inf")), t
        _ulp1(length, ln64)
        fin = torch.isfinite(lg64)
        _within("ray_sample logit", (logits.detach().cpu().double() - lg64)[fin].abs(), C_LOGIT * U * absw[fin])
        lg2, ln2, vd2 = ray_head.ray_sample(sigma, origin, points, frame, nw, step, with_gt)
        assert torch.equal(lg2, logits.detach()) and torch.equal(ln2, length) and torch.equal(vd2, valid), t
        if R == 0:
            continue
        # upstream gradient on every slot; on -inf slots also NaN and inf (zeroed by the wrapper's nan_to_num)
        g = torch.Generator().manual_seed(R + nw)
        gl = torch.randn(logits.shape, generator=g)
        gl[gl.abs() < 0.05] = 0.0
        inf_slot = lg64 == float("-inf")
        pick = torch.rand(logits.shape, generator=g)
        gl[inf_slot & (pick < 0.3)] = float("nan")
        gl[inf_slot & (pick > 0.7)] = float("inf")
        logits.backward(gl.to(cuda))
        sc = ref.sample_backward_fp64(c["sigma"], c["origin"], c["points"], c["frame"],
                                      torch.nan_to_num(gl, nan=0.0, posinf=0.0, neginf=0.0), nw, step, with_gt)
        _scatter_ok("ray_sample grad_sigma", s.grad, sc)


def check_ce(cuda, c, nw, step, tag):
    sigma, origin, points, frame = _dev(c, cuda)
    R, nf, Z, Y, X = _dims(c)
    dims = (R, nf, Z, Y, X, nw, step)
    out = [torch.full((R,), 7.0, device=cuda) for _ in range(3)]        # ce, lse, valid: every row is written
    _abi("ray_ce_forward", cuda, sigma, origin, points, frame, *out, *dims)
    ce, lse, valid = out
    o = ref.ce_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step)
    assert torch.equal(valid.cpu() > 0, o.valid), tag
    inv = ~o.valid
    assert (ce.cpu()[inv] == 0).all() and (lse.cpu()[inv] == 0).all(), tag
    _within("ray_ce ce", (ce.cpu().double() - o.ce)[o.valid].abs(), SAFETY * U * o.ce_cond[o.valid])
    _within("ray_ce lse", (lse.cpu().double() - o.lse)[o.valid].abs(), SAFETY * U * o.lse_cond[o.valid])
    again = [torch.empty(R, device=cuda) for _ in range(3)]
    _abi("ray_ce_forward", cuda, sigma, origin, points, frame, *again, *dims)
    assert all(torch.equal(a, b) for a, b in zip(again, out)), f"{tag}: ray_ce forward not deterministic"
    # rays whose only unmasked sample is the GT (origin far outside): ce = 0, and they scatter nothing
    only_gt = o.valid & c["far"] if "far" in c else torch.zeros(R, dtype=torch.bool)
    assert (ce.cpu()[only_gt] == 0).all(), tag
    if R == 0:
        return
    g = torch.Generator().manual_seed(R * 3 + nw)
    gce = torch.randn(R, generator=g)
    gce[torch.rand(R, generator=g) < 0.15] = 0.0                       # rays with grad_ce = 0 scatter nothing
    for gc, what in ((gce, "grad_ce"), (None, "grad_ce=nullptr")):
        gs = torch.zeros_like(sigma)
        _abi("ray_ce_backward", cuda, sigma, origin, points, frame, lse, None if gc is None else gc.to(cuda), gs,
             *dims)
        sc = ref.ce_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, gc).scatter
        _scatter_ok("ray_ce grad_sigma", gs, sc)
    for keep, what in ((torch.zeros(R, dtype=torch.bool), "grad_ce = 0"), (only_gt, "only the GT unmasked")):
        gs = torch.zeros_like(sigma)
        _abi("ray_ce_backward", cuda, sigma, origin, points, frame, lse, torch.where(keep, 1.0, 0.0).to(cuda),
             gs, *dims)
        assert not gs.any(), f"{tag}: {what} scattered"


def _noise(c, nw, step, seed):
    """Gumbel(0,1) noise, with exact ties planted where waypoints sample the constant block exactly."""
    R = c["points"].shape[0]
    g = torch.Generator().manual_seed(seed)
    noise = -torch.empty(R, nw).exponential_(generator=g).log()
    lg, *_ = ref.sample_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, True)
    ten = (lg[:, 1:] == 10.0) & _exact_rows(c, step)[:, None]
    tie = ten.sum(-1) >= 2
    noise[tie[:, None] & ten] = 20.0
    return noise.contiguous(), tie


def check_gumbel(cuda, c, nw, step, tag):
    sigma, origin, points, frame = _dev(c, cuda)
    R, nf, Z, Y, X = _dims(c)
    dims = (R, nf, Z, Y, X, nw, step)
    noise, tie = _noise(c, nw, step, R + 5 * nw)
    out = [torch.full((R,), 7.0, device=cuda) for _ in range(3)]
    _abi("ray_gumbel_forward", cuda, sigma, origin, points, frame, noise.to(cuda), *out, *dims)
    dist, lse, p = (t.cpu() for t in out)
    again = [torch.empty(R, device=cuda) for _ in range(3)]
    _abi("ray_gumbel_forward", cuda, sigma, origin, points, frame, noise.to(cuda), *again, *dims)
    assert all(torch.equal(a, b) for a, b in zip(again, out)), f"{tag}: ray_gumbel forward not deterministic"
    o = ref.gumbel_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, noise)
    _, ln, _, _ = ref.sample_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, True)
    ln = ln[:, 1:]
    assert not o.valid.logical_not().logical_and((dist != 0) | (lse != 0) | (p != 0)).any(), tag
    none = o.valid & o.dist.isnan()                 # every waypoint masked: the reference's softmax is NaN
    assert (dist[none] == ln[none, 0]).all() and (lse[none] == float("-inf")).all() and (p[none] == 0).all(), tag
    near = o.valid & ~none & (o.margin <= SAFETY * U * o.tie_cond) & ~_exact_rows(c, step)
    strict = o.valid & ~none & ~near
    assert torch.equal(dist[strict], o.dist[strict]), f"{tag}: gumbel dist"
    for r in near.nonzero().squeeze(-1).tolist():
        k = int((ln[r] == dist[r]).nonzero()[0])
        assert o.y[r, k] >= o.y[r, o.index[r]] - SAFETY * U * o.tie_cond[r], f"{tag} ray {r}: not a near tie"
        NEAR_TIES.append(f"gumbel {tag} ray {r}: kernel waypoint {k}, fp64 {int(o.index[r])}, margin {o.margin[r]:.2e}")
    _within("ray_gumbel lse", (lse.double() - o.lse)[strict].abs(), SAFETY * U * o.lse_cond[strict])
    _within("ray_gumbel p_next", (p.double() - o.p_next)[strict].abs(),
            SAFETY * U * (2 * o.lse_cond[strict] + 4) * o.p_next[strict] + nw * TINY)
    if tie.any():                                   # planted exact ties: the smallest waypoint index wins
        ten = (noise == 20.0) & tie[:, None]
        want = torch.where(ten, torch.arange(nw), nw).amin(-1)
        sel = tie & strict
        assert torch.equal(o.index[sel], want[sel]) and torch.equal(dist[sel], ln[sel].gather(1, want[sel, None])[:, 0])
    if R == 0:
        return
    g = torch.Generator().manual_seed(R + 9 * nw)
    gd = torch.randn(R, generator=g)
    gd[near] = 0.0
    gs = torch.zeros_like(sigma)
    _abi("ray_gumbel_backward", cuda, sigma, origin, points, frame, *out, gd.to(cuda), gs, *dims)
    sc = ref.gumbel_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, noise, gd).scatter
    _scatter_ok("ray_gumbel grad_sigma", gs, sc, extra=1)


def check_argmax(cuda, c, nw, step, tag):
    sigma, origin, points, frame = _dev(c, cuda)
    R, nf, Z, Y, X = _dims(c)
    dims = (R, nf, Z, Y, X, nw, step)
    depth, index = torch.full((R,), 7.0, device=cuda), torch.full((R,), 7.0, device=cuda)
    _abi("ray_argmax", cuda, sigma, origin, points, frame, depth, index, *dims)
    d2 = torch.full((R,), 7.0, device=cuda)
    _abi("ray_argmax", cuda, sigma, origin, points, frame, d2, None, *dims)
    assert torch.equal(d2, depth), f"{tag}: depth without index"
    d3, i3 = ray_head.ray_argmax(sigma, origin, points, frame, nw, step)
    assert torch.equal(d3, depth) and torch.equal(i3, index), f"{tag}: ray_argmax not deterministic"
    o = ref.argmax_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step)
    _, ln, _, _ = ref.sample_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step, False)
    idx, depth = index.cpu().long(), depth.cpu()
    f, live = ref.ray_frames(c["frame"], R, nf)
    assert (idx[~live] == 0).all() and (depth[~live] == 0).all(), tag
    assert torch.equal(depth[live], ln[live].gather(1, idx[live, None])[:, 0]), f"{tag}: depth is not its waypoint's"
    near = live & (o.margin <= SAFETY * U * 32 * o.absw) & ~_exact_rows(c, step)
    strict = ~near
    bad = strict & (idx != o.index)
    assert not bad.any(), f"{tag}: arg-max differs on {int(bad.sum())} rays, e.g. {bad.nonzero()[:5].tolist()}"
    for r in (near & (idx != o.index)).nonzero().squeeze(-1).tolist():
        assert o.value[r, idx[r]] >= o.value[r, o.index[r]] - SAFETY * U * 32 * o.absw[r], f"{tag} ray {r}: not a tie"
        NEAR_TIES.append(f"argmax {tag} ray {r}: kernel {int(idx[r])}, fp64 {int(o.index[r])}, margin {o.margin[r]:.2e}")


CHECKS = (check_sample, check_ce, check_gumbel, check_argmax)


# ---- the tests ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,nw", COMBOS, ids=[f"{n}-w{w}" for n, w in COMBOS])
@pytest.mark.parametrize("check", CHECKS, ids=[f.__name__[6:] for f in CHECKS])
def test_entry_point_vs_fp64(cuda, check, name, nw):
    check(cuda, case(name), nw, 1.0 if name.startswith("lattice") else STEP[nw], f"{name} w{nw}")


def test_case_hits_the_edges():
    """The inputs reach what they claim: exact-lattice samples, zero-weight outside corners, faces, ties."""
    c = case("lattice8x16x32")
    f, live = ref.ray_frames(c["frame"], c["points"].shape[0], 3)
    length, masked, coord, gin = ref.waypoints(c["origin"], c["points"], f, c["grid"], 64, 1.0, True)
    frac = coord - coord.floor()
    ok = live[:, None] & ~masked
    assert ((frac == 0).all(-1) & ok).any() and ((frac == 0.5).any(-1) & ok).any()
    idx, w = ref.corners(coord, c["grid"])
    assert ((idx < 0) & (w == 0) & ok[..., None]).any() and ((idx < 0) & (w > 0) & ok[..., None]).any()
    pts = c["points"]
    for a, size in enumerate((32, 16, 8)):
        on = live & ((pts[:, a] == 0) | (pts[:, a] == size))
        assert on.sum() == 2 and not gin[on].any()
    o = ref.argmax_fp64(c["sigma"], c["origin"], c["points"], c["frame"], 32, 1.0)
    ex = _exact_rows(c, 1.0)
    assert ex.sum() == 5 and (o.margin[ex] == 0).all() and (o.index[ex] == 4).all()      # exact ties, 8 lanes
    assert (live & (o.margin == float("inf")) & (o.index == 0)).any()      # all -inf: index 0
    for name in ("5x13x29", "z1"):
        lg, _, vd, _ = ref.sample_fp64(case(name)["sigma"], case(name)["origin"], case(name)["points"],
                                       case(name)["frame"], 64, 0.5, True)
        fr = case(name)["frame"]
        late = vd & (fr == 1) & torch.isinf(lg[:, 1]) & torch.isfinite(lg[:, 1:]).any(-1)
        never = vd & (fr == 2) & torch.isinf(lg[:, 1:]).all(-1)
        assert late.any() and never.any()


@pytest.mark.parametrize("R", [0, 1, 7, 8, 9])
def test_block_tail(cuda, R):
    c = dict(case("5x13x29"))
    rows = torch.randperm(c["points"].shape[0], generator=torch.Generator().manual_seed(R))[:R]
    for k in ("points", "frame", "exact", "far"):
        c[k] = c[k][rows].contiguous()
    for check in CHECKS:
        check(cuda, c, 33, 1.0, f"R{R}")


def test_frame_none(cuda):
    c = dict(case("lattice8x16x32"))
    c["frame"], c["far"] = None, torch.zeros(c["points"].shape[0], dtype=torch.bool)
    for check in CHECKS:
        check(cuda, c, 64, 0.5, "frame=None")


def test_sample_optional_outputs(cuda):
    c = case("5x13x29")
    sigma, origin, points, frame = _dev(c, cuda)
    R, nf, Z, Y, X = _dims(c)
    full = [torch.empty((R, 34), device=cuda), torch.empty((R, 34), device=cuda), torch.empty(R, device=cuda)]
    _abi("ray_sample", cuda, sigma, origin, points, frame, *full, R, nf, Z, Y, X, 33, 1.0, 1)
    for keep in range(3):
        part = [torch.full_like(t, 7.0) if i == keep else None for i, t in enumerate(full)]
        _abi("ray_sample", cuda, sigma, origin, points, frame, *part, R, nf, Z, Y, X, 33, 1.0, 1)
        assert torch.equal(part[keep], full[keep])


def test_full_size_ce_gradient_whole_volume(cuda):
    """3 frames of 16x200x200, 30 000 rays, 512 waypoints: ce, lse, valid and grad_sigma over the whole volume."""
    g = torch.Generator().manual_seed(0)
    R, nf, (Z, Y, X) = 30000, 3, (16, 200, 200)
    sigma = torch.randn(nf, Z, Y, X, generator=g)
    origin = torch.tensor([100.0, 100.0, 10.0]) + 0.5 * torch.randn(nf, 3, generator=g)
    ang = torch.rand(R, generator=g) * 6.2831853
    el = (torch.rand(R, generator=g) * 40 - 30) * 3.14159265 / 180
    rng = (2 + 68 * torch.rand(R, generator=g)) / 0.512
    frame = (torch.arange(R) * nf // R).to(torch.int32)
    d = torch.stack([el.cos() * ang.cos(), el.cos() * ang.sin(), el.sin() * 1.024], -1)
    pts = (origin[frame.long()] + d * rng[:, None]).contiguous()
    c = dict(sigma=sigma, origin=origin, points=pts, frame=frame, grid=(Z, Y, X))
    check_ce(cuda, c, 512, 1.0, "full size")


def test_argmax_nan_takes_the_first_nan(cuda):
    """torch's max returns a NaN's index: so does the kernel, whichever lane holds the NaN."""
    c = dict(case("lattice8x16x32"))
    sigma = c["sigma"].clone()
    o0 = lattice_origin(c["grid"])
    sigma[0, int(o0[2] - 0.5), int(o0[1] - 0.5), int(o0[0]) + 6] = float("nan")
    c["sigma"] = sigma
    for nw, step in ((32, 1.0), (64, 0.125)):
        o = ref.argmax_fp64(c["sigma"], c["origin"], c["points"], c["frame"], nw, step)
        nan_rows = o.margin.isinf() & (o.index > 0)
        assert nan_rows.any()
        check_argmax(cuda, c, nw, step, f"nan w{nw}")


def test_gumbel_takes_the_exact_argmax_not_the_softmax_one(cuda):
    """Two waypoint values of logit + noise one fp32 step apart round to the same softmax value: the reference's
    arg-max of softmax(logit + noise) takes the first, the kernel the larger (DESIGN.md 4.4)."""
    c = case("lattice8x16x32")
    o0 = lattice_origin(c["grid"])
    pts = torch.stack([o0 + torch.tensor([0.0, 0.0, 3.25])])                 # +z through the zero column
    nw = 8
    noise = torch.full((1, nw), -30.0)
    a = np.float32(0.1)
    noise[0, 0], noise[0, 1] = float(a), float(np.nextafter(a, np.float32(1)))
    lg, ln, vd, _ = ref.sample_fp64(c["sigma"], c["origin"], pts, torch.zeros(1, dtype=torch.int32), nw, 1.0, True)
    assert vd.all() and (lg[0, 1:3] == 0).all()
    y = (lg[0, 1:].float() + noise[0])
    soft = y.softmax(-1)
    assert soft[0] == soft[1] and int(soft.max(-1)[1]) == 0 and int(y.argmax()) == 1
    dist = ray_head.gumbel_distance(c["sigma"].to(cuda), c["origin"].to(cuda), pts.to(cuda),
                                    torch.zeros(1, dtype=torch.int32, device=cuda), nw, 1.0, noise.to(cuda))
    assert float(dist[0]) == float(ln[0, 2])


def test_host_wrappers_on_mixed_tindex(cuda):
    """get_grid_features, ce_regularization_loss and decode_ray_depth on tindex values that are frames, fractional,
    negative or >= F, against the oracle, in one call each."""
    base = case("5x13x29")
    bs, nf, nw, step = 2, 3, 33, 1.0
    lw = [[0.5, 1.0], [1.5, 2.0], [0.25, 3.0]]
    g = torch.Generator().manual_seed(4)
    sigma = [torch.randn(bs, nf, *base["grid"], generator=g) for _ in range(2)]
    origin = base["origin"][None].expand(bs, nf, 3).contiguous()
    M = base["points"].shape[0]
    gt = torch.stack([base["points"], base["points"].flip(0)]).contiguous()
    tindex = torch.randint(0, nf, (bs, M), generator=g).float()
    odd = torch.rand(bs, M, generator=g)
    tindex[odd < 0.1] = 0.5
    tindex[(odd >= 0.1) & (odd < 0.2)] = -1.0
    tindex[(odd >= 0.2) & (odd < 0.25)] = float(nf)
    tindex[(odd >= 0.25) & (odd < 0.3)] = nf + 1.5
    frame = torch.where((tindex >= 0) & (tindex < nf) & (tindex == tindex.floor()), tindex, -1.0).to(torch.int32)
    sg = [s.to(cuda).requires_grad_(True) for s in sigma]
    r_mask, r_feat, r_w, r_len = ray_head.get_grid_features(origin.to(cuda), gt.to(cuda), tindex.to(cuda), sg, lw,
                                                            step, nw)
    lgs, absws, lens, ws = [[], []], [[], []], [], []
    for b in range(bs):
        per = [ref.sample_fp64(s[b], origin[b], gt[b], frame[b], nw, step, True) for s in sigma]
        order = per[0][2].nonzero().squeeze(-1)
        order = order[torch.argsort(frame[b][order], stable=True)]            # frame-major, valid rows
        for lvl in range(2):
            lgs[lvl].append(per[lvl][0][order])
            absws[lvl].append(per[lvl][3][order])
        lens.append(per[0][1][order])
        ws.append(torch.tensor(lw)[frame[b][order].long()].t())
    lg64 = torch.stack([torch.cat(x, 0) for x in lgs])
    absw = torch.stack([torch.cat(x, 0) for x in absws])
    assert torch.equal(r_mask.cpu() == float("-inf"), lg64[0] == float("-inf"))
    fin = torch.isfinite(lg64)
    _within("get_grid_features logit", (r_feat.detach().cpu().double() - lg64)[fin].abs(), C_LOGIT * U * absw[fin])
    assert torch.equal(r_w.cpu(), torch.cat(ws, 1).float())
    _ulp1(r_len, torch.cat(lens, 0))
    # the fused CE loss and its gradient
    loss = ray_head.ce_regularization_loss(origin.to(cuda), gt.to(cuda), tindex.to(cuda), sg, lw, step, nw)
    loss.backward()
    lw64 = torch.tensor(lw, dtype=torch.float64)
    outs = [[ref.ce_fp64(s[b], origin[b], gt[b], frame[b], nw, step) for b in range(bs)] for s in sigma]
    wts = [[torch.where(outs[l][b].valid, lw64[frame[b].clamp(min=0).long(), l], 0.0) for b in range(bs)]
           for l in range(2)]
    den = sum(w.sum() for ww in wts for w in ww).clamp(min=1)
    num = sum((outs[l][b].ce * wts[l][b]).sum() for l in range(2) for b in range(bs))
    n = sum(int(o.valid.sum()) for oo in outs for o in oo)
    depth = math.ceil(math.log2(n)) + 16        # the device sums reduce in a tree over a few serial steps
    bound = SAFETY * U * sum(((outs[l][b].ce_cond + depth * outs[l][b].ce.abs()) * wts[l][b]).sum()
                             for l in range(2) for b in range(bs)) / den
    _within("ce_regularization_loss", (loss.detach().cpu().double() - num / den).abs(), bound)
    for l in range(2):
        for b in range(bs):
            sc = ref.ce_fp64(sigma[l][b], origin[b], gt[b], frame[b], nw, step, wts[l][b] / den).scatter
            _scatter_ok("ce_regularization_loss grad", sg[l].grad[b], sc, extra=2)
    # decode
    for b in range(bs):
        pred, gdist = ray_head.decode_ray_depth(sigma[1][b].to(cuda), origin[b].to(cuda), gt[b].to(cuda),
                                                tindex[b].to(cuda), step, nw)
        o = ref.argmax_fp64(sigma[1][b], origin[b], gt[b], frame[b], nw, step)
        live = frame[b] >= 0
        assert (pred.cpu()[~live] == 0).all() and (gdist.cpu()[~live] == 0).all()
        strict = live & ~(o.margin <= SAFETY * U * 32 * o.absw)
        assert torch.equal(pred.cpu()[strict], o.depth[strict])
        _, ln, _, _ = ref.sample_fp64(sigma[1][b], origin[b], gt[b], frame[b], nw, step, True)
        np.testing.assert_array_max_ulp(gdist.cpu()[live].numpy(), ln[live, 0].numpy(), maxulp=2)
