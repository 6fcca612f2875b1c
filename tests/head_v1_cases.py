"""Seeded cases for the ViDARHeadV1 loss / decode goldens (tools/make_golden_head_v1.py and the tests).

The shipped structure (vidar_1_8_nusc_3future.py): history_queue_length 4, 3 history + current + 1 future head
frame, per-frame weights (0.2, 0.4, 0.6, 1.0, 1.2), a 5-entry loss_weight with its trailing [0]; here on a small
grid with ragged GT lists, random rigid frame transforms and some points outside the volume."""
import numpy as np
import torch

BEV_H, BEV_W, Z = 16, 16, 8
PC_RANGE = [-24.0, -24.0, -4.0, 24.0, 24.0, 4.0]       # 3 m x 3 m x 1 m voxels
INTER, BS = 2, 2
HISTORY_QUEUE_LENGTH = 4
N_FRAMES = 9                                           # GT / transform frames 0 .. 8
RAY_GRID_NUM, RAY_GRID_STEP = 24, 1.0
LOSS_W = [[1.0], [0.9], [0.8], [0.7], [0.0]]
HEAD_KW = dict(history_queue_length=HISTORY_QUEUE_LENGTH, pred_history_frame_num=3, pred_future_frame_num=1,
               per_frame_loss_weight=(0.2, 0.4, 0.6, 1.0, 1.2), ray_grid_num=RAY_GRID_NUM,
               ray_grid_step=RAY_GRID_STEP, use_ce_loss=True, use_dist_loss=False, use_dense_loss=True,
               dense_loss_weight=0.5, eval_within_grid=False)
HEAD_FRAMES = 5
CALL_KW = dict(start_idx=0, tgt_bev_h=BEV_H, tgt_bev_w=BEV_W, tgt_pc_range=PC_RANGE)
CASES = {
    "shipped": dict(valid_frames=[0, 1, 2, 3], full_prev_bev_exists=True),
    "no_prev_bev": dict(valid_frames=[0, 1, 2, 3], full_prev_bev_exists=False),
    "valid_0_2": dict(valid_frames=[0, 2], full_prev_bev_exists=True),
}
# The reference draws the same Gumbel noise for 'no_prev_bev' as for 'shipped' (same seed, same shapes), and its
# gradient is the 'shipped' gradient of the current head frame alone; the golden keeps one copy of each
# (tools/make_golden_head_v1.py checks both when it writes them).
SAME_DRAWS = {"no_prev_bev": "shipped"}


def weighted_frames(name, idx):
    """Frames of loss index `idx` whose dense term has a non-zero weight: the only ones whose Gumbel noise can
    change a loss or a gradient, and the only noise the golden stores."""
    phf = HEAD_KW["pred_history_frame_num"]
    i = idx if CASES[name]["full_prev_bev_exists"] else phf
    if idx != i or HEAD_KW["per_frame_loss_weight"][i] == 0:
        return []
    if i != phf:
        return [0]
    return [t for t in range(len(CASES[name]["valid_frames"])) if LOSS_W[t][0] != 0]


def _rigid(g):
    """Row-vector 4x4 transform (x' = [x 1] @ T): a rotation of a few degrees and a shift of a few metres."""
    ang = np.radians(np.array([2.0, 2.0, 6.0])) * (2 * torch.rand(3, generator=g).numpy() - 1)
    cx, cy, cz = np.cos(ang)
    sx, sy, sz = np.sin(ang)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = (rz @ ry @ rx).T
    T[3, :3] = np.array([3.0, 3.0, 0.3]) * (2 * torch.rand(3, generator=g).numpy() - 1)
    return T


def case(name, seed=0, bs=BS):
    g = torch.Generator().manual_seed(seed)
    valid_frames = CASES[name]["valid_frames"]
    V = len(valid_frames)
    preds = torch.randn(V, INTER, HEAD_FRAMES, bs, BEV_H * BEV_W, Z, generator=g)
    lo = torch.tensor([-26.0, -26.0, -4.5])
    hi = torch.tensor([26.0, 26.0, 4.5])
    gt_points, img_metas = [], []
    for b in range(bs):
        n = 500 + 70 * b                                             # ragged
        xyz = lo + (hi - lo) * torch.rand(n, 3, generator=g)         # a few outside the volume
        extra = torch.rand(n, 1, generator=g)                        # intensity column
        t = torch.randint(0, N_FRAMES, (n, 1), generator=g).float()
        gt_points.append(torch.cat([xyz, extra, t], 1))
        cur2ref = np.stack([_rigid(g) for _ in range(N_FRAMES)])
        img_metas.append(dict(total_cur2ref_lidar_transform=cur2ref,
                              total_ref2cur_lidar_transform=np.linalg.inv(cur2ref)))
    pred_dict = dict(next_bev_preds=preds, valid_frames=valid_frames,
                     full_prev_bev_exists=CASES[name]["full_prev_bev_exists"])
    return dict(pred_dict=pred_dict, gt_points=gt_points, img_metas=img_metas, loss_weight=np.array(LOSS_W))
