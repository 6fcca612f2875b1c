"""The cases of test_nn_sort_scale_gpu.py reach the edges they are built for, on both H100 SM counts: candidate
splits with several tiles, exact ties across splits / across tiles / inside one tile, sort keys spanning chunks,
keys only in the last chunk or in none, and the counting sort's 33+ and 64 key histograms."""
import numpy as np
import pytest

from tests import nn_sort_cases as nc


def _verified_kinds(ties, cands, keep, queries, Lc_of, splits):
    """Kinds of the planted ties whose two candidates really are among the first fp32 minima of their query."""
    kinds = set()
    for key, i, a, b in ties:
        m = nc.first_minima(queries(key)[i], cands(key), None if keep is None else keep(key))
        if a in m and b in m:
            kinds.add(nc.tie_kind(a, b, Lc_of(key), splits))
    return kinds


@pytest.mark.parametrize("sms", nc.SM_COUNTS)
def test_segmented_case_splits_and_ties(sms):
    c = nc.segments_case(sms)
    Lc = np.diff(c["c_off"])
    assert c["splits"] >= 2
    assert max(nc.split_chunk(int(n), c["splits"]) for n in Lc) > nc.NN_TILE      # >= 2 tiles in one split
    seg = lambda a, off: (lambda s: a[off[s]:off[s + 1]])
    kinds = _verified_kinds(c["ties"], seg(c["c"], c["c_off"]), seg(c["c_mask"], c["c_off"]),
                            seg(c["q"], c["q_off"]), lambda s: int(Lc[s]), c["splits"])
    assert kinds == {"split", "tile", "same"}, kinds
    assert len(c["ties"]) >= 300
    # masked queries, a segment without candidates, one with every candidate masked, one without queries
    assert (c["q_mask"] == 0).any() and (Lc == 0).any() and (np.diff(c["q_off"]) == 0).any()
    s = nc.ALL_MASKED
    assert Lc[s] > 0 and not c["c_mask"][c["c_off"][s]:c["c_off"][s + 1]].any()


@pytest.mark.parametrize("sms", nc.SM_COUNTS)
def test_batched_case_splits_and_ties(sms):
    c = nc.knn_case(3, sms)
    L2 = c["len2"]
    assert c["splits"] >= 2 and nc.split_chunk(int(L2[0]), c["splits"]) > nc.NN_TILE
    assert (L2 == 0).any() and (c["len1"] < nc.KNN_P1).any() and (L2 % nc.NN_TILE != 0).any()
    kinds = _verified_kinds(c["ties"], lambda n: c["p2"][n, :L2[n]], None, lambda n: c["p1"][n],
                            lambda n: int(L2[n]), c["splits"])
    assert kinds == {"split", "tile", "same"}, kinds
    # the crowd sharing one nearest candidate
    crowd = c["p1"][0, -400:]
    assert all(nc.first_minima(q, c["p2"][0])[0] == 5 for q in crowd[::37])


def _key_chunks(keys, key):
    return set((np.nonzero(keys == key)[0] // nc.SORT_CHUNK).tolist())


def test_sort_cases_reach_chunk_edges_and_key_counts():
    Ms = {m for _, _, m in nc.ALIGN_CASES.values()} | {m for _, m, _ in nc.DECODE_CASES.values()}
    assert {1023, 1024, 1025} <= Ms
    assert any(nc.sort_chunks(m) >= 3 and m % nc.SORT_CHUNK for m in Ms)
    nkeys = [v for _, v, _ in nc.ALIGN_CASES.values()] + [f for f, _, _ in nc.DECODE_CASES.values()]
    assert any(33 <= k < 64 for k in nkeys) and 64 in nkeys     # histogram 32 * keys > 1024 threads; the limit

    spans = 0
    for name, (H, V, M) in nc.ALIGN_CASES.items():
        c = nc.align_case(name)
        last = nc.sort_chunks(M) - 1
        frames = c["gt"][0, :, 4]
        assert _key_chunks(frames, nc.LAST_ONLY) == {last}
        assert not (c["gt"][..., 4] == nc.NOWHERE).any()
        assert all(nc.LAST_ONLY in row and nc.NOWHERE in row for row in c["jobs"].tolist())
        assert all(len(set(r) - {-1}) == len([v for v in r if v >= 0]) for r in c["jobs"].tolist())
        assert np.isnan(c["gt"][1, -1]).all()
        spans = max(spans, max(len(_key_chunks(frames, f)) for f in c["jobs"][0] if f >= 0))
    assert spans >= 3

    for name, (F, M, _) in nc.DECODE_CASES.items():
        c = nc.decode_case(name)
        t = c["tindex"]
        assert (t == np.float32(0.5) + np.floor(t)).any() and (t < 0).any() and (t >= F).any()
        if F > 2:
            last = nc.sort_chunks(M) - 1
            assert all(_key_chunks(t[b], F - 1) == {last} for b in range(t.shape[0]))
            assert not (t == F - 2).any()
        # rows at the origin of their frame: gt_dist == 0
        f = np.clip(t, 0, F - 1).astype(np.int64)
        at = (c["rays"] == np.take_along_axis(c["origin_vox"], f[..., None], 1)).all(-1) & (t == f)
        assert at.sum() >= 20
