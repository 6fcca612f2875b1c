"""CPU oracle for the nearest-neighbour / Chamfer op.  TEST INFRASTRUCTURE.

numpy restatement of third_lib/chamfer_dist/chamferdist/chamferdist/knn_cpu.cpp:7-106 for K = 1
(squared distance summed over d in order, first strictly-smaller candidate wins) and of
ChamferDistance.forward (chamfer.py:20-133).  Pinned against the reference's own CPU build
(oracle/_ref/ref_knn_cpu.so = ext.cpp + knn_cpu.cpp compiled unmodified, and the reference
chamfer.py running on top of it): tests/golden/knn.npz via tools/make_golden_knn.py."""
import numpy as np


def nn(p1, p2, len1=None, len2=None, block=2048):
    """p1 [N,P1,D], p2 [N,P2,D] float32 -> dists [N,P1] float32, idx [N,P1] int64 (zero padded)."""
    p1, p2 = np.asarray(p1, np.float32), np.asarray(p2, np.float32)
    N, P1, D = p1.shape
    P2 = p2.shape[1]
    dists = np.zeros((N, P1), np.float32)
    idx = np.zeros((N, P1), np.int64)
    for n in range(N):
        l1 = P1 if len1 is None else int(len1[n])
        l2 = P2 if len2 is None else int(len2[n])
        if l2 == 0:
            continue
        for s in range(0, l1, block):
            a = p1[n, s:min(l1, s + block)]
            d = np.zeros((a.shape[0], l2), np.float32)
            for k in range(D):                                   # same accumulation order, fp32
                diff = a[:, None, k] - p2[n, None, :l2, k]
                d = d + diff * diff
            j = d.argmin(1)                                       # first minimum
            idx[n, s:s + a.shape[0]] = j
            dists[n, s:s + a.shape[0]] = d[np.arange(a.shape[0]), j]
    return dists, idx


def nn_backward(p1, p2, idx, grad_dists, len1=None, len2=None):
    p1, p2 = np.asarray(p1, np.float32), np.asarray(p2, np.float32)
    N, P1, D = p1.shape
    g1 = np.zeros_like(p1)
    g2 = np.zeros_like(p2, dtype=np.float64)
    for n in range(N):
        l1 = P1 if len1 is None else int(len1[n])
        if len2 is not None and int(len2[n]) == 0:                # no candidate: no gradient
            continue
        j = idx[n, :l1]
        diff = 2.0 * grad_dists[n, :l1, None] * (p1[n, :l1] - p2[n, j])
        g1[n, :l1] = diff
        np.add.at(g2[n], j, -diff.astype(np.float64))
    return g1, g2.astype(np.float32)


def chamfer(source, target, bidirectional=False, reverse=False, reduction="mean"):
    f_d, f_i = nn(source, target)
    cf = f_d.sum(1)
    cb = None
    if reverse or bidirectional:
        b_d, b_i = nn(target, source)
        cb = b_d.sum(1)
    red = {"sum": np.sum, "mean": np.mean, None: lambda x: x}[reduction]
    if bidirectional:
        return red(cf), red(cb)
    if reverse:
        return red(cb)
    return red(cf)
