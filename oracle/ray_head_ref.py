"""CPU oracle for the ViDAR head ray sampler / CE loss / arg-max decode.  TEST INFRASTRUCTURE.

Restates projects/mmdet3d_plugin/bevformer/dense_heads/vidar_head_base.py
  _get_grid_features :420-509, the CE branch of loss :586-592, and the decode loop of
  get_point_cloud_prediction :700-734
with plain torch ops (F.grid_sample for the trilinear interpolation, as the reference does).
Pinned by tests/golden/ray_head.npz, produced by running the reference's own methods in this
container (tools/make_golden_ray_head.py).

The second half is an fp64 oracle of the same operations (`sample_fp64`, `ce_fp64`, `gumbel_fp64`,
`argmax_fp64`), for judging the CUDA kernels by fp32 error bounds rather than by an fp32 restatement.
The waypoints, their lengths, the boundary mask and the un-normalised grid_sample coordinates are the
reference's fp32 statements, one torch fp32 op each (no contraction), so the same voxel corners are
picked; from those coordinates on everything is fp64: corner weights, an explicit 8-corner gather,
log-sum-exp, softmax and closed-form gradients.  Alongside each value the oracle returns the magnitudes
the test tolerances are built from: per sample sum_j |sigma_j w_j|, and per voxel of every backward the
scatter volumes of `Scatter`.
"""
from collections import namedtuple

import torch
import torch.nn.functional as F


def sample_frame(sigma_f, origin, gt, num_way, step, with_gt=True):
    """One frame.  sigma_f [Z,Y,X]; origin [3]; gt [R,3] (voxel units).
    -> logits [R,K] (-inf where masked), length [R,K], valid [R] bool."""
    Z, Y, X = sigma_f.shape
    o = origin.view(1, 1, 3)
    ray = gt - origin.view(1, 3)
    unit = ray / torch.sqrt((ray ** 2).sum(-1, keepdim=True))
    t = (torch.arange(num_way, dtype=torch.float64) + 0.5).to(gt.dtype) * step
    pts = o + unit.unsqueeze(1) * t.view(1, -1, 1)
    if with_gt:
        pts = torch.cat([gt.unsqueeze(1), pts], 1)
    length = torch.sqrt(((pts - o) ** 2).sum(-1))
    size = torch.tensor([X, Y, Z], dtype=gt.dtype)
    norm = pts / size * 2 - 1
    masked = ((norm <= -1.) | (norm >= 1)).any(-1)
    valid = ((norm[:, 0] > -1.) & (norm[:, 0] < 1.)).all(-1) if with_gt else torch.ones(len(gt), dtype=torch.bool)
    val = F.grid_sample(sigma_f.view(1, 1, Z, Y, X), norm.view(1, 1, *norm.shape), mode="bilinear",
                        padding_mode="zeros", align_corners=False).view(norm.shape[:2])
    logits = val + torch.zeros_like(val).masked_fill(masked, float("-inf"))
    return logits, length, valid


def grid_features(origin_grids, gt_grids, gt_tindex, intermediate_sigma, loss_weights, step, num_way):
    """All four outputs of _get_grid_features for lists over (batch, frame)."""
    bs, Fr = intermediate_sigma[0].shape[:2]
    masks, feats, weights, lengths = [], [], [], []
    for b in range(bs):
        for f in range(Fr):
            gt = gt_grids[b][gt_tindex[b] == f]
            per_lvl, keep, length = [], None, None
            for sig in intermediate_sigma:
                logits, length, keep = sample_frame(sig[b, f], origin_grids[b, f], gt, num_way, step)
                per_lvl.append(logits[keep])
            feats.append(torch.stack(per_lvl, 0))
            lengths.append(length[keep])
            masks.append(torch.isinf(per_lvl[0]))
            w = torch.stack([torch.full((int(keep.sum()),), float(loss_weights[f][l]))
                             for l in range(len(intermediate_sigma))], 0)
            weights.append(w)
    mask = torch.cat(masks, 0)
    r_mask = torch.zeros(mask.shape).masked_fill(mask, float("-inf"))
    return r_mask, torch.cat(feats, 1), torch.cat(weights, 1), torch.cat(lengths, 0)


def ce_loss(r_feat_total, r_loss_weight_total):
    """loss :586-592 -- cross entropy with label 0 over the K logits of every ray."""
    logp0 = torch.log_softmax(r_feat_total, -1)[..., 0]
    return (-(logp0) * r_loss_weight_total).sum() / torch.clamp(r_loss_weight_total.sum(), min=1)


def decode_frame(sigma_f, origin, gt, num_way, step):
    """get_point_cloud_prediction :712-732 for one frame -> (pred_dist [R], argmax index [R])."""
    logits, length, _ = sample_frame(sigma_f, origin, gt, num_way, step, with_gt=False)
    Z, Y, X = sigma_f.shape
    # the decode path applies no boundary mask: outside samples are exact zeros -> -inf
    o = origin.view(1, 1, 3)
    ray = gt - origin.view(1, 3)
    unit = ray / torch.sqrt((ray ** 2).sum(-1, keepdim=True))
    t = (torch.arange(num_way, dtype=torch.float64) + 0.5).to(gt.dtype) * step
    pts = o + unit.unsqueeze(1) * t.view(1, -1, 1)
    norm = pts / torch.tensor([X, Y, Z], dtype=gt.dtype) * 2 - 1
    val = F.grid_sample(sigma_f.view(1, 1, Z, Y, X), norm.view(1, 1, *norm.shape), mode="bilinear",
                        padding_mode="zeros", align_corners=False).view(norm.shape[:2])
    val = val.masked_fill(val == 0, float("-inf"))
    idx = val.max(1)[1]
    return torch.gather(length, 1, idx.view(-1, 1)).squeeze(-1), idx


# ---- fp64 oracle of the csrc/ray_head.cu entry points -------------------------------------------------
U32 = 2.0 ** -24            # unit roundoff of fp32 round-to-nearest
FLUSH = 2.0 ** -126 / U32   # in units of U32: an exp or product below fp32's smallest normal may flush to 0
CHUNK_SAMPLES = 1 << 19     # rays x samples per chunk: ~70 MB of corner indices and weights

Chunk = namedtuple("Chunk", "rows f live length masked gt_inside idx w logit absw")
Scatter = namedtuple("Scatter", "grad mag err count")
Scatter.__doc__ = """fp64 [F, Z, Y, X] volumes of one backward: grad = sum of the contributions c = dl_k w_j;
mag = sum |c|; err = sum eps_k w_j, eps_k a bound on the fp32 error of dl_k in units of U32; count = number of
contributions.  An fp32 kernel scattering the same contributions with red.add lands within
U32 * (err + (count + 6) * mag) of grad, to first order: 6 roundings in w_j and dl_k w_j, and at most count - 1
roundings of a partial sum no larger than mag."""
CEResult = namedtuple("CEResult", "ce lse valid lse_cond ce_cond scatter")
GumbelResult = namedtuple("GumbelResult", "dist lse p_next valid index margin tie_cond lse_cond y scatter")
ArgmaxResult = namedtuple("ArgmaxResult", "index depth margin absw value")


def _f32(v):
    return torch.tensor(v, dtype=torch.float32)


def _div(a, b):
    """Correctly rounded fp32 a / b (through fp64: one rounding of an exact-enough quotient)."""
    return (a.double() / b.double()).float()


def _norm3(d):
    """sqrt((d0 d0 + d1 d1) + d2 d2), one fp32 op per step, the kernels' summation order.  The square root is
    taken through fp64 because torch's vectorised fp32 sqrt on the CPU is not always correctly rounded."""
    return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).double().sqrt().float()


def ray_frames(frame, R, num_frames):
    """(frame as int64, live): frame None means frame 0; a row of a frame outside [0, F) is skipped."""
    f = torch.zeros(R, dtype=torch.long) if frame is None else frame.long()
    return f, (f >= 0) & (f < num_frames)


def waypoints(origin, points, f, grid, num_way, step, with_gt):
    """The fp32 statements of _get_grid_features for rays of frame f (clamped into range: the callers ignore
    rows of no frame).  grid = (Z, Y, X).  -> length [R,K], masked [R,K], un-normalised grid_sample coordinates
    [R,K,3] (x, y, z), gt_inside [R]; K = num_way + with_gt, sample 0 the GT point when with_gt."""
    Z, Y, X = grid
    o = origin.float()[f.clamp(0, origin.shape[0] - 1)]
    g = points.float()
    ray = g - o
    unit = _div(ray, _norm3(ray)[:, None])
    t = (torch.arange(num_way, dtype=torch.float64) + 0.5).float() * _f32(step)
    pts = o[:, None, :] + unit[:, None, :] * t[None, :, None]
    if with_gt:
        pts = torch.cat([g[:, None, :], pts], 1)
    length = _norm3(pts - o[:, None, :])
    size = torch.tensor([X, Y, Z], dtype=torch.float32)
    two, one = _f32(2.0), _f32(1.0)
    norm = _div(pts, size) * two - one
    masked = ((norm <= -1) | (norm >= 1)).any(-1)
    coord = ((norm + one) * size - one) / two
    ng = _div(g, size) * two - one
    gt_inside = ((ng > -1) & (ng < 1)).all(-1)
    return length, masked, coord, gt_inside


_BITS = torch.tensor([[j & 1, (j >> 1) & 1, j >> 2] for j in range(8)])     # grid_sample's corner order


def corners(coord, grid):
    """Trilinear corners of un-normalised coordinates [..., 3] (x, y, z) on a [Z, Y, X] volume: index [..., 8]
    (z, y, x row-major, -1 for a corner outside the volume: grid_sample's zero padding) and fp64 weight [..., 8].
    The weights are computed exactly from the fp32 coordinates, up to one fp64 rounding per product."""
    Z, Y, X = grid
    c = coord.double()
    lo = torch.floor(c)
    w1, w0 = c - lo, (lo + 1) - c
    base = torch.nan_to_num(lo, nan=-2.0, posinf=-2.0, neginf=-2.0).long()
    p = base[..., None, :] + _BITS                                  # [..., 8, 3]
    w = torch.where(_BITS == 1, w1[..., None, :], w0[..., None, :]).prod(-1)
    xs, ys, zs = p[..., 0], p[..., 1], p[..., 2]
    inside = (xs >= 0) & (xs < X) & (ys >= 0) & (ys < Y) & (zs >= 0) & (zs < Z)
    return torch.where(inside, (zs * Y + ys) * X + xs, -1), w


def _chunks(sigma, origin, points, frame, num_way, step, with_gt, need_gt_inside=False):
    """Per chunk of rays: geometry, corners and the fp64 trilinear value of every sample (masked or not).  Only
    live rows are visited, and with need_gt_inside only those whose GT point lies inside the volume: the callers
    leave the other rows at their initial values."""
    nf, Z, Y, X = sigma.shape
    vol = sigma.detach().double().reshape(nf, -1)
    R = points.shape[0]
    f_all, live_all = ray_frames(frame, R, nf)
    keep = live_all
    if need_gt_inside:
        keep = keep & waypoints(origin, points, f_all, (Z, Y, X), 0, 1.0, False)[3]
    todo = keep.nonzero().squeeze(-1)
    K = num_way + int(bool(with_gt))
    rows = max(1, CHUNK_SAMPLES // K)
    for a in range(0, todo.numel(), rows):
        sl = todo[a:a + rows]
        f = f_all[sl]
        length, masked, coord, gin = waypoints(origin, points[sl], f, (Z, Y, X), num_way, step, with_gt)
        idx, w = corners(coord, (Z, Y, X))
        v = vol[f.clamp(0, nf - 1)[:, None, None], idx.clamp(min=0)]
        terms = torch.where(idx >= 0, v, 0.0) * w            # an outside corner adds an exact zero
        yield Chunk(sl, f, live_all[sl], length, masked, gin, idx, w, terms.sum(-1), terms.abs().sum(-1))


class _ScatterAcc:
    def __init__(self, shape):
        self.shape, self.n = tuple(shape), shape[1] * shape[2] * shape[3]
        self.vols = [torch.zeros(shape[0] * self.n, dtype=torch.float64) for _ in range(4)]

    def add(self, c, dl, eps, take):
        """dl, eps [Rc, K] fp64 for the samples `take` [Rc, K] of chunk c."""
        sel = take[..., None] & (c.idx >= 0)
        gi = (c.f.clamp(min=0)[:, None, None] * self.n + c.idx)[sel]
        contrib = (dl[..., None] * c.w)[sel]
        for vol, val in zip(self.vols, (contrib, contrib.abs(), (eps[..., None] * c.w)[sel], torch.ones_like(contrib))):
            vol.index_add_(0, gi, val)

    def result(self):
        return Scatter(*(v.view(self.shape) for v in self.vols))


def lse_cond(absw_max, v_max, K, lse):
    """First-order bound, in units of U32, on the fp32 error of an online log-sum-exp over K trilinear logits, and
    on the relative error of each exp(v_k - lse): 16 A per logit (A = max_k sum_j |sigma_j w_j|) for the logit,
    the running max and the final max; per online step, expf's 2 ulp and the rounding of its argument
    (|v - m| <= 2 V, V = max |v_k|) over K/32 lane steps and 5 shuffle levels; log and the final add."""
    return 48 * absw_max + (2 * v_max + 8) * (K / 32 + 8) + 2 * lse.abs()


def sample_fp64(sigma, origin, points, frame, num_way, step, with_gt):
    """vidar_ray_sample in fp64.  sigma [F,Z,Y,X], origin [F,3], points [R,3], frame int [R] or None; a row of a
    frame outside [0, F) gives -inf logits, zero lengths and valid 0.  -> logits [R,K] fp64 (-inf where masked),
    length [R,K] fp32, valid [R] bool, absw [R,K] fp64 = sum_j |sigma_j w_j| (0 where masked)."""
    K, R = num_way + int(bool(with_gt)), points.shape[0]
    logits = torch.full((R, K), float("-inf"), dtype=torch.float64)
    length = torch.zeros((R, K), dtype=torch.float32)
    valid = torch.zeros(R, dtype=torch.bool)
    absw = torch.zeros((R, K), dtype=torch.float64)
    for c in _chunks(sigma, origin, points, frame, num_way, step, with_gt):
        ok = c.live[:, None] & ~c.masked
        logits[c.rows] = torch.where(ok, c.logit, float("-inf"))
        length[c.rows] = torch.where(c.live[:, None], c.length, 0.0)
        valid[c.rows] = c.live & (c.gt_inside if with_gt else True)
        absw[c.rows] = torch.where(ok, c.absw, 0.0)
    return logits, length, valid, absw


def sample_backward_fp64(sigma, origin, points, frame, grad_logits, num_way, step, with_gt):
    """vidar_ray_sample_backward in fp64: grad_logits [R,K] (finite, as the kernel receives them) scattered
    through the corner weights of every unmasked sample of a live row -> Scatter (sigma gives the shape)."""
    acc = _ScatterAcc(sigma.shape)
    gl = grad_logits.double()
    for c in _chunks(sigma, origin, points, frame, num_way, step, with_gt):
        g = gl[c.rows]
        acc.add(c, g, torch.zeros_like(g), c.live[:, None] & ~c.masked & (g != 0))
    return acc.result()


def ce_fp64(sigma, origin, points, frame, num_way, step, grad_ce=None):
    """vidar_ray_ce_forward / backward in fp64: cross entropy with label 0 over the GT slot and num_way
    waypoints; rows of no frame or with the GT outside the volume give ce = lse = 0, valid 0 and scatter
    nothing.  grad_ce [R] (None = 1) -> CEResult: ce, lse [R] fp64, valid [R] bool, lse_cond / ce_cond [R] (error
    bounds in units of U32, see lse_cond), scatter (d sum(grad_ce * ce) / d sigma)."""
    R, K = points.shape[0], num_way + 1
    ce, lse_all = torch.zeros(R, dtype=torch.float64), torch.zeros(R, dtype=torch.float64)
    valid = torch.zeros(R, dtype=torch.bool)
    lcond, ccond = torch.zeros(R, dtype=torch.float64), torch.zeros(R, dtype=torch.float64)
    g_all = torch.ones(R, dtype=torch.float64) if grad_ce is None else grad_ce.double()
    acc = _ScatterAcc(sigma.shape)
    onehot = torch.zeros(K, dtype=torch.float64)
    onehot[0] = 1
    for c in _chunks(sigma, origin, points, frame, num_way, step, True, need_gt_inside=True):
        ok = c.live & c.gt_inside
        lg = torch.where(c.masked, float("-inf"), c.logit)
        lse = torch.logsumexp(lg, -1)
        lse = torch.where(ok, lse, 0.0)
        p = torch.exp(lg - lse[:, None])
        lam = lse_cond(torch.where(c.masked, 0.0, c.absw).amax(-1), torch.where(c.masked, 0.0, c.logit.abs()).amax(-1),
                       K, lse)
        ce_r = torch.where(ok, lse - c.logit[:, 0], 0.0)
        ce[c.rows], lse_all[c.rows], valid[c.rows] = ce_r, lse, ok
        lcond[c.rows] = torch.where(ok, lam, 0.0)
        ccond[c.rows] = torch.where(ok, lam + 16 * c.absw[:, 0] + ce_r.abs(), 0.0)
        g = g_all[c.rows]
        dl = g[:, None] * (p - onehot)
        eps = g.abs()[:, None] * (p * lam[:, None] + 2 * (p - onehot).abs() + FLUSH)
        acc.add(c, dl, eps, (ok & (g != 0))[:, None] & ~c.masked)
    return CEResult(ce, lse_all, valid, lcond, ccond, acc.result())


def gumbel_fp64(sigma, origin, points, frame, num_way, step, noise, grad_dist=None):
    """vidar_ray_gumbel_forward / backward in fp64, by the statements of _custom_gumbel_softmax_distance
    (vidar_head_base.py:754-773) on the waypoint logits (the GT slot dropped) with the arg-max taken over
    logit + noise (first index on ties).  Rows of no frame or with the GT outside give zeros.  A row whose
    waypoints are all masked gives what the reference's softmax gives: NaN dist, lse and p_next.
    -> GumbelResult: dist [R] fp32, lse, p_next [R] fp64, valid [R], index [R] (waypoint, 0-based), margin [R]
    (best minus second-best logit + noise, inf when fewer than two are finite), tie_cond [R] (bound on the fp32
    error of a difference of two logit + noise values, units of U32), lse_cond [R], y [R, num_way] (logit + noise,
    -inf where masked), scatter of
    d sum(grad_dist * dist) / d sigma through p_next (grad_dist None = 1)."""
    R = points.shape[0]
    nz = noise.double()
    dist = torch.zeros(R, dtype=torch.float32)
    lse_all, p_all = torch.zeros(R, dtype=torch.float64), torch.zeros(R, dtype=torch.float64)
    valid, index = torch.zeros(R, dtype=torch.bool), torch.zeros(R, dtype=torch.long)
    margin, tcond, lcond = (torch.zeros(R, dtype=torch.float64) for _ in range(3))
    y_all = torch.full((R, num_way), float("-inf"), dtype=torch.float64)
    g_all = torch.ones(R, dtype=torch.float64) if grad_dist is None else grad_dist.double()
    acc = _ScatterAcc(sigma.shape)
    for c in _chunks(sigma, origin, points, frame, num_way, step, True, need_gt_inside=True):
        ok = c.live & c.gt_inside
        masked, length, absw = c.masked[:, 1:], c.length[:, 1:], torch.where(c.masked, 0.0, c.absw)[:, 1:]
        lg = torch.where(masked, float("-inf"), c.logit[:, 1:])
        y = lg + nz[c.rows]
        idx = y.argmax(-1)
        pred = length.gather(1, idx[:, None])[:, 0]
        mx = lg.amax(-1)
        e = torch.exp(lg - mx[:, None])
        whole = e.sum(-1)
        later = length > pred[:, None]
        p = (e * later).sum(-1) / whole
        lse = mx + torch.log(whole)
        if num_way > 1:
            top = y.topk(2, -1).values
            m = torch.where(top[:, 1] == float("-inf"), float("inf"), top[:, 0] - top[:, 1])
        else:
            m = torch.full((y.shape[0],), float("inf"), dtype=torch.float64)
        lam = lse_cond(absw.amax(-1), torch.where(masked, 0.0, lg.abs()).amax(-1), num_way, lse)
        dist[c.rows] = torch.where(ok, torch.where(mx == float("-inf"), float("nan"), pred), 0.0)
        lse_all[c.rows], p_all[c.rows] = torch.where(ok, lse, 0.0), torch.where(ok, p, 0.0)
        valid[c.rows], index[c.rows] = ok, torch.where(ok, idx, 0)
        margin[c.rows] = torch.where(ok, m, float("inf"))
        y_all[c.rows] = y
        tcond[c.rows] = torch.where(ok, 32 * absw.amax(-1) + 2 * y.amax(-1).abs().nan_to_num(0.0, 0.0, 0.0) + 2, 0.0)
        lcond[c.rows] = torch.where(ok, lam, 0.0)
        gd = g_all[c.rows] * pred.double()
        sm = torch.where(masked, 0.0, e / whole[:, None])
        dl = gd[:, None] * sm * (later.double() - p[:, None])
        eps = gd.abs()[:, None] * (sm * (2 * lam[:, None] + 6) + FLUSH)
        gt_slot = torch.zeros_like(dl[:, :1])                          # the GT slot scatters nothing
        acc.add(c, torch.cat([gt_slot, dl], 1), torch.cat([gt_slot, eps], 1),
                torch.cat([gt_slot.bool(), (ok & (gd != 0))[:, None] & ~masked], 1))
    return GumbelResult(dist, lse_all, p_all, valid, index, margin, tcond, lcond, y_all, acc.result())


def argmax_fp64(sigma, origin, points, frame, num_way, step):
    """vidar_ray_argmax in fp64, by the statements of get_point_cloud_prediction (:712-732): the waypoints'
    trilinear values without the boundary mask, exact zeros -> -inf, torch's max (the first NaN, else the first
    maximum; all -inf -> 0), that waypoint's length.  Rows of no frame give index 0 and depth 0.
    -> ArgmaxResult: index [R], depth [R] fp32, margin [R] (best minus second-best value, inf when fewer than two
    are finite or the row holds a NaN), absw [R] (max over the waypoints of sum_j |sigma_j w_j|), value [R, num_way]
    (the values compared, -inf for rows of no frame)."""
    R = points.shape[0]
    index, depth = torch.zeros(R, dtype=torch.long), torch.zeros(R, dtype=torch.float32)
    margin, absw = torch.full((R,), float("inf"), dtype=torch.float64), torch.zeros(R, dtype=torch.float64)
    value = torch.full((R, num_way), float("-inf"), dtype=torch.float64)
    for c in _chunks(sigma, origin, points, frame, num_way, step, False):
        v = torch.where(c.logit == 0, float("-inf"), c.logit)
        nan = v.isnan()
        num = torch.where(nan, float("-inf"), v)
        idx = torch.where(nan.any(-1), nan.double().argmax(-1), num.argmax(-1))
        if num_way > 1:
            top = num.topk(2, -1).values
            m = torch.where((top[:, 1] == float("-inf")) | nan.any(-1), float("inf"), top[:, 0] - top[:, 1])
        else:
            m = torch.full((v.shape[0],), float("inf"), dtype=torch.float64)
        index[c.rows] = torch.where(c.live, idx, 0)
        depth[c.rows] = torch.where(c.live, c.length.gather(1, idx[:, None])[:, 0], 0.0)
        margin[c.rows] = torch.where(c.live, m, float("inf"))
        absw[c.rows] = torch.where(c.live, c.absw.amax(-1), 0.0)
        value[c.rows] = v
    return ArgmaxResult(index, depth, margin, absw, value)
