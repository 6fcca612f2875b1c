"""The point pipeline's host half and its oracle, without a GPU: the oracle (oracle/point_pipeline_ref.py) on the
plans recorded by vidar_b200.point_pipeline's transforms equals the reference's own statements
(tests/golden/point_pipeline.npz) bit for bit in every case; the transforms leave numpy's generator where the
reference's leave it after every call; the index-vector shuffles make the reference's 2-D shuffles; unsupported
settings raise."""
import numpy as np
import pytest

from oracle import point_pipeline_ref as ref
from tests import point_pipeline_cases as cases
from vidar_b200 import point_pipeline as pp

Z, METAS = cases.golden()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("meta", METAS, ids=[m["name"] for m in METAS])
def test_oracle_equals_golden(meta, tmp_path):
    gathered, _ = cases.replay(Z, meta, str(tmp_path))
    got = ref.gather([pp.frame_plan(r) for r in gathered], meta["ego_mask"])
    want = Z[f"{meta['name']}.gt"]
    assert got.shape == want.shape
    assert np.array_equal(bits(got), bits(want))
    padded = ref.gather([pp.frame_plan(r) for r in gathered], meta["ego_mask"], padded=True)
    assert np.array_equal(bits(padded[~np.isnan(padded[:, 0])]), bits(want))


@pytest.mark.parametrize("meta", METAS, ids=[m["name"] for m in METAS])
def test_numpy_state_after_every_call(meta, tmp_path):
    _, states = cases.replay(Z, meta, str(tmp_path))
    want_k, want_g = Z[f"{meta['name']}.states"], Z[f"{meta['name']}.gauss"]
    assert len(states) == len(want_k)
    for i, (k, g) in enumerate(states):
        assert np.array_equal(k, want_k[i]), f"call {i}"
        assert g == want_g[i], f"call {i}"


def test_golden_covers_the_cases():
    z = {m["name"]: Z[f"{m['name']}.gt"] for m in METAS}
    assert z["hard_nonzero"].shape == (0, 5)
    assert z["max_voxels"].shape[0] <= 150
    q = z["queue3"]
    assert set(np.unique(q[:, 4]).tolist()) == {0.0, 2.0}           # frame 1 has no survivors
    assert all(np.isfinite(v).all() for v in z.values())


@pytest.mark.parametrize("n,aliased", [(0, True), (1, True), (2, False), (1000, True), (1000, False), (5, False)])
def test_index_shuffles_equal_2d_shuffles(n, aliased):
    rng = np.random.default_rng(n)
    pts = rng.normal(size=(n, 5)).astype(np.float32)
    n_prev = 0 if aliased else 37
    np.random.seed(11)
    cur = pts.copy()
    prev = cur if aliased else rng.normal(size=(n_prev, 5)).astype(np.float32)
    np.random.shuffle(cur)
    np.random.shuffle(prev)
    st_ref = np.random.get_state()
    np.random.seed(11)
    idx = np.arange(n, dtype=np.int32)
    np.random.shuffle(idx)
    if aliased:
        np.random.shuffle(idx)
    else:
        np.random.shuffle(np.arange(n_prev, dtype=np.int32))
    st = np.random.get_state()
    assert np.array_equal(bits(pts[idx]), bits(cur))
    assert np.array_equal(st[1], st_ref[1]) and st[2:] == st_ref[2:]


def test_argument_validation():
    with pytest.raises(ValueError):
        pp.LoadPointsFromFile(coord_type="LIDAR", load_dim=5, use_dim=4)
    with pytest.raises(ValueError):
        pp.LoadPointsFromFile(coord_type="LIDAR", load_dim=6, use_dim=5)
    pp.LoadPointsFromFile(coord_type="LIDAR", load_dim=5, use_dim=[0, 1, 2, 3, 4])
    with pytest.raises(ValueError):
        pp.CustomLoadPointsFromMultiSweeps(sweeps_num=2)                       # default use_dim [0, 1, 2, 4]
    with pytest.raises(ValueError):
        pp.CustomLoadPointsFromMultiSweeps(use_dim=5, file_client_args=dict(backend="petrel"))
    cfg = dict(max_num_points=1, point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], voxel_size=[1, 1, 1])
    with pytest.raises(ValueError):
        pp.CustomVoxelBasedPointSampler(dict(cfg, max_num_points=2), time_dim=4)
    with pytest.raises(ValueError):
        pp.CustomVoxelBasedPointSampler(cfg, prev_sweep_cfg=cfg, time_dim=4)
    with pytest.raises(ValueError):
        pp.CustomVoxelBasedPointSampler(cfg, time_dim=3)
    with pytest.raises(ValueError):
        pp.CustomVoxelBasedPointSampler(dict(cfg, voxel_size=[0.01, 0.01, 0.01]), time_dim=4)
    with pytest.raises(ValueError):
        pp.CustomVoxelBasedPointSampler(cfg, time_dim=4)(dict(points=np.zeros((3, 5), np.float32)))
    with pytest.raises(ValueError):
        pp.pack([dict(points=np.zeros((3, 4), np.float32))], None)
    with pytest.raises(RuntimeError):
        pp.gather_gt_points([dict(points=np.zeros((3, 5), np.float32))], None, "cpu")


def test_config_pipelines_match_the_config():
    load, sweeps, sampler = pp.config_train_pipeline()
    assert (sweeps.sweeps_num, sweeps.pad_empty_sweeps, sweeps.remove_close, sweeps.hard_sweeps_timestamp,
            sweeps.random_select) == (2, True, True, 0, False)
    assert sampler.grid == (102, 102, 8) and sampler.max_voxels == 50000
    assert len(pp.config_test_pipeline()) == 1


def test_upload_is_raw_points_and_int32_orders(tmp_path):
    meta = METAS[0]
    gathered, _ = cases.replay(Z, meta, str(tmp_path))
    raw, perm = pp.upload_bytes(gathered)
    plan = pp.frame_plan(gathered[0])
    assert raw == sum(s.raw.nbytes for s in {id(s.raw): s for s in plan.current()}.values())
    assert perm == plan.perm.nbytes
