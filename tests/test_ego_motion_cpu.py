"""Ego motion on the host (vidar_b200/ego_motion.py): the queue metas, the encoder's shift and the decoder's
previous-frame grids against tests/golden/ego_motion.npz, written by tools/make_golden_ego_motion.py from the
reference's own get_data_info, union2one, get_bev_features and _align_bev_coordnates statements; and the option's
contract: the default graph is unchanged, missing poses and the row-sharded encoder are rejected."""
import os

import numpy as np
import pytest
import torch

from vidar_b200 import ego_motion as ego
from vidar_b200 import pretrain, synthetic

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ego_motion.npz")
CASES = [(4, 3), (4, 6), (4, 3)]                  # (image frames, future frames) of the golden's cases


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _queue(g, c):
    T, F = CASES[c]
    queue = []
    for t in range(T + F):
        f = {k: g[f"c{c}.in{t}.{k}"] for k in ("ego2global_translation", "ego2global_rotation",
                                                "lidar2ego_translation", "lidar2ego_rotation", "can_bus")}
        f = {k: (v if k == "can_bus" else [float(x) for x in v]) for k, v in f.items()}
        f["scene_token"] = f"scene-{int(g[f'c{c}.in{t}.scene'])}"
        if t < T:
            f["img_filename"] = []
        queue.append(f)
    return queue


@pytest.mark.parametrize("c", range(len(CASES)))
def test_queue_metas_equal_the_reference_bit_for_bit(golden, c):
    T, _ = CASES[c]
    metas = ego.queue_metas(_queue(golden, c))
    assert len(metas) == T
    for t in range(T):
        for k in ("can_bus", "lidar2global_rotation", "ref_lidar_to_cur_lidar"):
            np.testing.assert_array_equal(metas[t][k], golden[f"c{c}.m{t}.{k}"], err_msg=f"frame {t} {k}")
        assert metas[t]["prev_bev_exists"] == bool(golden[f"c{c}.m{t}.prev_bev_exists"])
    for k in ("future_can_bus", "future2ref_lidar_transform", "ref2future_lidar_transform",
              "total_cur2ref_lidar_transform", "total_ref2cur_lidar_transform"):
        np.testing.assert_array_equal(metas[-1][k], golden[f"c{c}.cur.{k}"], err_msg=k)


def test_scene_change_cuts_the_history(golden):
    metas = ego.queue_metas(_queue(golden, 2))
    assert [m["prev_bev_exists"] for m in metas] == [False, True, False, True]
    assert not metas[2]["can_bus"][[0, 1, 2, 17]].any()


@pytest.mark.parametrize("c", range(len(CASES)))
@pytest.mark.parametrize("hw", [200, 50])
def test_shift_and_angle_equal_the_reference(golden, c, hw):
    metas = ego.queue_metas(_queue(golden, c))
    for t, m in enumerate(metas):
        shift = ego.bev_shift([m], hw, hw).astype(np.float32)          # uploaded as fp32, as new_tensor casts
        np.testing.assert_array_equal(shift, golden[f"c{c}.m{t}.shift{hw}"])
        assert m["can_bus"][-1] == golden[f"c{c}.m{t}.can_bus"][-1]       # the rotation angle in degrees


@pytest.mark.parametrize("c", range(len(CASES)))
def test_future_grids_match_the_reference(golden, c):
    _, F = CASES[c]
    metas = ego.queue_metas(_queue(golden, c))
    f2r, r2h = ego.future_matrices([metas[-1]], F)
    mats = torch.matmul(torch.from_numpy(f2r).float(), torch.from_numpy(r2h).float())
    for k in range(1, F + 1):
        ref = ego.future_grids(mats[k - 1], 50, 50, pretrain.PC_RANGE)             # [1, Q, 1, 2]
        np.testing.assert_allclose(ref.numpy(), golden[f"c{c}.ref{k}"], rtol=0, atol=2e-6)
        tgt = pretrain.bev_geometry.get_reference_points(50, 50, dim="2d", device="cpu")[:, :, 0]
        np.testing.assert_array_equal(tgt.numpy(), golden[f"c{c}.tgt{k}"])


def test_restated_quaternion_is_a_rotation():
    q = ego.Quaternion(synthetic.LIDAR2EGO_ROTATION)
    R = q.rotation_matrix
    np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-15)
    assert abs(np.linalg.det(R) - 1) < 1e-15
    yaw = np.deg2rad(30.0)
    assert abs(ego.quaternion_yaw(ego.Quaternion([np.cos(yaw / 2), 0, 0, np.sin(yaw / 2)])) - yaw) < 1e-15


def test_missing_pose_key_is_named():
    queue = pretrain.synthetic_queue(2, 1, (32, 32), 1, 100, poses=True)
    del queue[1]["lidar2ego_rotation"]
    with pytest.raises(ValueError, match="lidar2ego_rotation"):
        ego.queue_metas(queue)
    with pytest.raises(ValueError, match="prev_bev_exists"):
        ego.require_metas([dict(can_bus=np.zeros(18))])


def test_default_queue_and_sample_unchanged():
    a = pretrain.synthetic_queue(2, 1, (32, 32), 1, 100, seed=3)
    b = pretrain.synthetic_queue(2, 1, (32, 32), 1, 100, seed=3, poses=True)
    assert all(set(x) < set(y) for x, y in zip(a, b))
    assert not any(k in f for f in a for k in ego.POSE_KEYS)
    assert "pose_metas" not in pretrain.synthetic_sample("cpu", frames=2, cams=1, img_hw=(32, 32), rays_per_frame=10,
                                                         future_frames=1, bev_hw=(8, 8))


def _small(**kw):
    return pretrain.SyntheticViDAR(num_cams=1, encoder_layers=2, decoder_layers=1, future_frames=1, history_frames=1,
                                   latent_layer=1, bev_hw=(8, 8), ray_grid_num=16, **kw)


def test_state_dict_unchanged_by_default_and_only_the_future_can_bus_mlp_under_the_option():
    torch.manual_seed(0)
    base = {k: tuple(v.shape) for k, v in _small().state_dict().items()}
    ego_sd = {k: tuple(v.shape) for k, v in _small(ego_motion=True).state_dict().items()}
    assert base.keys() == ego_sd.keys()
    assert {k for k in base if base[k] != ego_sd[k]} == {"future_can_bus_mlp.0.weight"}
    assert ego_sd["future_can_bus_mlp.0.weight"] == (128, 4)
    assert not _small().ego_motion
    assert all("ego_motion" not in cfg for cfg in pretrain.CONFIGS.values())


def test_row_sharded_encoder_rejects_ego_motion():
    with pytest.raises(ValueError, match="row-sharded"):
        _small(ego_motion=True).set_process_group(None, row_sharded=True)


def test_drive_is_nuscenes_like():
    d = synthetic.drive(20, seed=5)
    pos = np.array([f["ego2global_translation"] for f in d])
    speed = np.linalg.norm(np.diff(pos, axis=0), axis=1) / 0.5
    assert speed.max() <= 15 + 1e-9
    yaw = np.array([ego.quaternion_yaw(ego.Quaternion(f["ego2global_rotation"])) for f in d])
    rate = np.rad2deg(np.abs(np.angle(np.exp(1j * np.diff(yaw))))) / 0.5
    assert rate.max() <= 10 + 1e-6
    assert len({f["scene_token"] for f in synthetic.drive(6, 0, scene_change=3)}) == 2


def test_first_future_angle_is_relative_to_the_current_frames_absolute_yaw():
    """_prepare_data_info makes the current frame's results dict once per queue, so union2one's future loop starts
    from the current frame's absolute can_bus, not from the history loop's deltas."""
    drive = synthetic.drive(7, 0)
    metas = ego.queue_metas([dict(f, img_filename=()) for f in drive[:4]] + drive[4:])
    absolute = [ego.frame_can_bus(f)["can_bus"][-1] for f in drive[3:]]
    np.testing.assert_array_equal(metas[-1]["future_can_bus"][1:, -1], np.diff(absolute))
    assert abs(metas[-1]["future_can_bus"][1, -1]) < 10
