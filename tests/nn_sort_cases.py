"""Seeded cases for the nearest-neighbour search (csrc/knn.cu) and the stable counting sort (csrc/counting_sort.cuh)
at training sizes, with exact ties and key changes placed on the kernels' split, tile and chunk boundaries.

The launch arithmetic below mirrors knn.cu (`vidar_nn_forward`, `vidar_nn_segments_forward`) and the sort's chunking;
the builders use it only to place ties and keys, and every case also scatters a few hundred duplicate pairs at random
indices, so the cases keep reaching a split boundary if the split heuristic changes.  No CUDA here: the CPU test
(test_nn_sort_cases_cpu.py) checks that the cases reach the edges they are built for."""
import numpy as np

NN_THREADS = 256          # queries per block of the search
NN_TILE = 1024            # candidates per shared-memory tile
SORT_CHUNK = 1024         # rows per block of the counting sort
SM_COUNTS = (114, 132)    # H100 PCIe and SXM


def cdiv(a, b):
    return -(-a // b)


def nn_splits(max_q, max_c, segments, sms):
    """Candidate splits of one query block (blockIdx.y): ~4 waves of (block, split) pairs, at least one tile each.
    For the batched search `segments` is the batch size N and max_q / max_c are P1 / P2."""
    bx = cdiv(max_q, NN_THREADS)
    return max(1, min(cdiv(4 * sms, bx * segments), cdiv(max_c, NN_TILE)))


def split_chunk(Lc, splits):
    return cdiv(Lc, splits)


def place(j, Lc, splits):
    """(split, tile within the split) that scans candidate j of a segment of Lc candidates."""
    chunk = split_chunk(Lc, splits)
    s = j // chunk
    return s, (j - s * chunk) // NN_TILE


def tie_kind(a, b, Lc, splits):
    """'split', 'tile' or 'same' (tile) for two candidates a, b of one segment."""
    (sa, ta), (sb, tb) = place(a, Lc, splits), place(b, Lc, splits)
    return "split" if sa != sb else ("tile" if ta != tb else "same")


def sort_chunks(M):
    return cdiv(M, SORT_CHUNK)


def boundary_pairs(Lc, splits):
    """Candidate index pairs (a, b), a < b, straddling every split boundary, the first tile boundary inside each
    split, and a pair inside one tile of the first split."""
    chunk = split_chunk(Lc, splits)
    out = []
    for s in range(splits):
        j0, j1 = s * chunk, min(Lc, (s + 1) * chunk)
        if j0 >= j1:
            break
        if s > 0:
            out.append((j0 - 1, j0))
        if j1 - j0 > NN_TILE:
            out.append((j0 + NN_TILE - 1, j0 + NN_TILE))
    if Lc >= 40:
        out.append((3, min(Lc, NN_TILE, chunk) - 2))
    return out


# ------------------------------------------------------------------ planting ties
def _plant(q, c, pairs, qrows, rng, offset_scale):
    """For each (a, b): candidate b := candidate a (bit-identical distance to every query) and query row qrows[k]
    := candidate a plus a small offset, so a / b are its nearest candidates.  Returns [(query row, a, b)]."""
    D = c.shape[1]
    out = []
    for (a, b), i in zip(pairs, qrows):
        c[b] = c[a]
        q[i] = c[a] + (offset_scale * (rng.random(D) - 0.5)).astype(np.float32)
        out.append((int(i), int(a), int(b)))
    return out


def _cloud(rng, n, D, lattice, ext=100.0):
    if lattice:                                   # small integers: distinct candidates at equal fp32 distances
        return rng.integers(0, 12, size=(n, D)).astype(np.float32)
    return (ext * rng.random((n, D))).astype(np.float32)


def _tie_rows(rng, Lq, used, k):
    free = np.setdiff1d(np.arange(Lq), np.asarray(sorted(used), dtype=np.int64))
    return rng.choice(free, size=k, replace=False)


def _plant_segment(rng, q, c, Lq, Lc, splits, n_random=300):
    """Boundary ties plus n_random duplicate pairs at random indices of one (query, candidate) segment."""
    if Lq == 0 or Lc < 2:
        return []
    pairs = boundary_pairs(Lc, splits)
    while len(pairs) < len(boundary_pairs(Lc, splits)) + n_random:
        a, b = sorted(rng.choice(Lc, 2, replace=False))
        pairs.append((int(a), int(b)))
    # every candidate in at most one pair, so a later copy cannot undo an earlier one
    seen, uniq = set(), []
    for a, b in pairs:
        if a not in seen and b not in seen:
            uniq.append((a, b))
            seen.update((a, b))
    uniq = uniq[:Lq]
    return _plant(q, c, uniq, _tie_rows(rng, Lq, set(), len(uniq)), rng, 0.2)


# ------------------------------------------------------------------ §2 batched search (chamfer.knn_points)
KNN_N, KNN_P1, KNN_P2 = 3, 4000, 16000
# element 0 full; element 1 no candidates and fewer queries; element 2 ragged, L2 not a multiple of 1024, lattice
KNN_L1 = (KNN_P1, 2900, 3700)
KNN_L2 = (KNN_P2, 0, 9077)


def knn_case(D, sms, seed=0):
    """p1 [N, P1, D], p2 [N, P2, D], len1, len2 int64, grad [N, P1] and the planted ties [(n, query, a, b)].
    Element 0 also has 400 queries sharing one nearest candidate (the backward's scatter)."""
    rng = np.random.default_rng(1000 * D + seed)
    N, P1, P2 = KNN_N, KNN_P1, KNN_P2
    splits = nn_splits(P1, P2, N, sms)
    p1 = np.zeros((N, P1, D), np.float32)
    p2 = np.zeros((N, P2, D), np.float32)
    ties = []
    for n in range(N):
        lattice = n == 2
        p1[n] = _cloud(rng, P1, D, lattice)
        p2[n] = _cloud(rng, P2, D, lattice)
        if lattice:                               # rows past the lengths hold junk the kernel must not read
            p1[n, KNN_L1[n]:] = 1e6
            p2[n, KNN_L2[n]:] = -1e6
        L1, L2 = KNN_L1[n], KNN_L2[n]             # the kernel sizes the splits by P2, each element splits its L2
        ties += [(n, i, a, b) for i, a, b in _plant_segment(rng, p1[n], p2[n], L1, L2, splits)]
    # a crowd of queries around candidate 5 of element 0, far from everything else
    p2[0, 5] = np.float32(-50.0)
    p1[0, P1 - 400:] = (np.float32(-50.0) + 0.5 * rng.random((400, D))).astype(np.float32)
    ties = [t for t in ties if not (t[0] == 0 and (t[1] >= P1 - 400 or 5 in t[2:]))]
    grad = rng.standard_normal((N, P1)).astype(np.float32)
    return dict(p1=p1, p2=p2, len1=np.array(KNN_L1, np.int64), len2=np.array(KNN_L2, np.int64), grad=grad,
                ties=ties, splits=splits)


# ------------------------------------------------------------------ §3 segmented search (vidar_nn_segments_forward)
# (queries, candidates, lattice) of each segment: a long one, one without candidates, one whose candidates are all
# masked, one without queries, a lattice one, a short one
SEGMENTS = ((3000, 12000, False), (500, 0, False), (700, 900, False), (0, 400, False), (2600, 7777, True),
            (1200, 3000, False))
ALL_MASKED = 2


def segments_case(sms, seed=0):
    """Flat q [Pq, 3], c [Pc, 3], offsets [S+1], uint8 masks and the planted ties [(segment, query, a, b)]
    (a, b within the segment)."""
    rng = np.random.default_rng(77 + seed)
    Lq = np.array([s[0] for s in SEGMENTS])
    Lc = np.array([s[1] for s in SEGMENTS])
    S = len(SEGMENTS)
    splits = nn_splits(int(Lq.max()), int(Lc.max()), S, sms)
    q_off = np.concatenate([[0], np.cumsum(Lq)]).astype(np.int64)
    c_off = np.concatenate([[0], np.cumsum(Lc)]).astype(np.int64)
    q = np.zeros((q_off[-1], 3), np.float32)
    c = np.zeros((c_off[-1], 3), np.float32)
    q_mask = (rng.random(q_off[-1]) > 0.1).astype(np.uint8)
    c_mask = (rng.random(c_off[-1]) > 0.1).astype(np.uint8)
    ties = []
    for s, (nq, nc, lattice) in enumerate(SEGMENTS):
        qs, cs = q[q_off[s]:q_off[s + 1]], c[c_off[s]:c_off[s + 1]]
        qs[:] = _cloud(rng, nq, 3, lattice)
        cs[:] = _cloud(rng, nc, 3, lattice)
        if s == ALL_MASKED:
            c_mask[c_off[s]:c_off[s + 1]] = 0
            continue
        for i, a, b in _plant_segment(rng, qs, cs, nq, nc, splits):
            q_mask[q_off[s] + i] = 1
            c_mask[c_off[s] + a] = c_mask[c_off[s] + b] = 1
            ties.append((s, i, a, b))
    return dict(q=q, c=c, q_off=q_off, c_off=c_off, q_mask=q_mask, c_mask=c_mask, ties=ties, splits=splits,
                max_q=int(Lq.max()), max_c=int(Lc.max()))


def first_minima(q, c, keep=None):
    """Indices of every candidate at the fp32 minimum squared distance of query q (summed in d order), first first."""
    d = np.zeros(len(c), np.float32)
    for k in range(c.shape[1]):
        diff = q[k] - c[:, k]
        d = d + diff * diff
    if keep is not None:
        d = np.where(keep.astype(bool), d, np.float32(np.inf))
    return np.nonzero(d == d.min())[0]


# ------------------------------------------------------------------ §4 counting sort users
ALIGN_CASES = {          # (head frames H, slots V, rows M)
    "h5_v51_m1025": (5, 51, 1025),
    "h5_v51_m20000": (5, 51, 20000),
    "h4_v64_m1025": (4, 64, 1025),
    "h4_v64_m20000": (4, 64, 20000),
}
ALIGN_VOXEL = [-51.2, -51.2, -5.0, 1.0 / 102.4, 1.0 / 102.4, 1.0 / 8.0, 200.0, 200.0, 16.0]
LAST_ONLY, NOWHERE = 500, 501    # frames of rows only in the last chunk / of no row


def _rigid(rng):
    ang = np.radians([3.0, 3.0, 20.0]) * (2 * rng.random(3) - 1)
    cx, cy, cz = np.cos(ang)
    sx, sy, sz = np.sin(ang)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = (rz @ ry @ rx).T
    T[3, :3] = np.array([5.0, 5.0, 0.5]) * (2 * rng.random(3) - 1)
    return T.astype(np.float32)


def align_case(name, bs=2, seed=0):
    """gt [bs, M, 5] (xyz, intensity, frame) with frames in shuffled order, sample 1 NaN-padded past 70 % of M;
    jobs [H, V] source frames (distinct per head frame, some -1, LAST_ONLY and NOWHERE in every head frame);
    mats [H*V, bs, 4, 4] random rigid transforms."""
    H, V, M = ALIGN_CASES[name]
    rng = np.random.default_rng(seed + M + V)
    n_frames = V + 10                            # some frames belong to no slot
    gt = np.empty((bs, M, 5), np.float32)
    gt[..., :3] = (rng.random((bs, M, 3)) * [100.0, 100.0, 8.0] - [50.0, 50.0, 4.0]).astype(np.float32)
    gt[..., 3] = rng.random((bs, M))
    gt[..., 4] = rng.integers(0, n_frames, (bs, M))
    last0 = (sort_chunks(M) - 1) * SORT_CHUNK
    gt[:, last0 + (M - last0) // 2:, 4] = LAST_ONLY
    gt[1, int(0.7 * M):] = np.nan
    jobs = np.full((H, V), -1, np.int64)
    for i in range(H):
        frames = rng.permutation(n_frames)[:V - 2]
        frames[rng.random(V - 2) < 0.05] = -1
        jobs[i, :V - 2] = frames
        jobs[i, V - 2:] = rng.permutation([LAST_ONLY, NOWHERE])
        jobs[i] = jobs[i, rng.permutation(V)]
    mats = np.stack([np.stack([_rigid(rng) for _ in range(bs)]) for _ in range(H * V)])
    return dict(gt=gt, jobs=jobs, mats=mats, voxel=np.float32(ALIGN_VOXEL))


DECODE_CASES = {          # (frames F, rows M, within_grid)
    "f3_m1023": (3, 1023, False),
    "f64_m1024": (64, 1024, True),
    "f3_m1025": (3, 1025, True),
    "f64_m1025": (64, 1025, False),
    "f64_m40000": (64, 40000, False),
    "f3_m40000_within": (3, 40000, True),
}
DECODE_PC = [-40.0, -40.0, -3.0, 40.0, 40.0, 3.0]
DECODE_SCALE = 80.0 / 160.0


def decode_case(name, bs=2, seed=0):
    """Inputs of ray_head.decode_clouds: tindex with frames in shuffled order, non-integer and out-of-range values,
    rows at their frame's origin (gt_dist == 0); with 64 frames one frame only in the last chunk and one in none."""
    F, M, within = DECODE_CASES[name]
    rng = np.random.default_rng(seed + 3 * M + F)
    origin_vox = (rng.random((bs, F, 3)) * [20.0, 20.0, 2.0] + [70.0, 70.0, 5.0]).astype(np.float32)
    origin = ((origin_vox - [80.0, 80.0, 6.0]) * np.float32(DECODE_SCALE)).astype(np.float32)
    rays = (rng.random((bs, M, 3)) * [170.0, 170.0, 14.0] - [5.0, 5.0, 1.0]).astype(np.float32)
    points = ((rays - [80.0, 80.0, 6.0]) * np.float32(DECODE_SCALE)).astype(np.float32)
    depth = (rng.random((bs, M)) * 60.0).astype(np.float32)
    t = rng.integers(-1, F + 2, (bs, M)).astype(np.float32)
    t[rng.random((bs, M)) < 0.05] += np.float32(0.5)
    if F > 2:
        last0 = (sort_chunks(M) - 1) * SORT_CHUNK
        t[t == F - 1] = 0
        t[:, last0 + (M - last0) // 2:] = F - 1                         # frame F-1: only in the last chunk
        t[t == F - 2] = 0                                               # frame F-2: in no chunk
    for b in range(bs):                                                 # rows at the origin of their frame
        at = rng.choice(M, 20, replace=False)
        f = np.clip(t[b, at], 0, F - 1).astype(np.int64)
        if F > 2:
            f[f >= F - 2] = 0
        t[b, at] = f
        rays[b, at] = origin_vox[b, f]
    return dict(depth=depth, rays=rays, points=points, tindex=t, origin_vox=origin_vox, origin=origin,
                scale=DECODE_SCALE, within_grid=within, pc_range=DECODE_PC)


# ------------------------------------------------------------------ dense Chamfer
DENSE_GRID = (100, 100, 16)


def dense_case(bs, F, R0=2500, M=12000, sms=132, seed=0):
    """dense_chamfer_loss inputs (dist [bs, F*R0], points, origin [bs, F, 3], gt [bs, M, 3], tindex [bs, M]) with
    duplicated pred rays (same end point and dist) on the candidate split / tile boundaries of the pred segments and
    a GT row next to each copy, and GT rows duplicated across sort chunk boundaries."""
    rng = np.random.default_rng(seed + 10 * bs + F)
    W, H, Z = DENSE_GRID
    ext = np.array([W, H, Z], np.float32)
    origin = (ext / 2 + rng.standard_normal((bs, F, 3))).astype(np.float32)
    ends = (2 + rng.random((bs, F * R0, 3)) * (ext - 4)).astype(np.float32)     # ray end points inside the box
    points = (ext / 2 + 3 * rng.standard_normal((bs, F * R0, 3))).astype(np.float32)
    dist = (40.0 * rng.random((bs, F * R0))).astype(np.float32)
    dist[rng.random((bs, F * R0)) < 0.1] = 0.0
    gt = (rng.random((bs, M, 3)) * (ext + 2) - 1).astype(np.float32)
    tindex = rng.integers(-1, F + 1, (bs, M)).astype(np.float32)
    max_len = max(R0, M)
    splits = nn_splits(max_len, max_len, 2 * bs * F, sms)
    pairs = boundary_pairs(R0, splits)
    pairs += [tuple(sorted(rng.choice(R0, 2, replace=False))) for _ in range(40)]
    for b in range(bs):
        gi = 0
        for f in range(F):
            o = origin[b, f]
            for a, c in pairs:
                for k in (a, c):                  # ray end == `ends`, so pred = (ends - o) * 0.1 up to rounding
                    points[b, f * R0 + k] = ends[b, f * R0 + a]
                    r = ends[b, f * R0 + a] - o
                    dist[b, f * R0 + k] = np.sqrt((r * r).sum())
                if gi < M:                        # a GT row of this pair beside the copies
                    gt[b, gi] = ends[b, f * R0 + a] + np.float32(0.3)
                    tindex[b, gi] = f
                    gi += 1
    for b in range(bs):                           # GT rows duplicated across the sort's chunk boundaries
        for c0 in range(SORT_CHUNK, M, SORT_CHUNK):
            gt[b, c0] = gt[b, c0 - 1]
            tindex[b, c0] = tindex[b, c0 - 1]
    return dict(dist=dist, points=points, origin=origin, gt=gt, gt_tindex=tindex, splits=splits, pairs=pairs)
