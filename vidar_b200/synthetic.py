"""Seeded synthetic workloads of the hot path (SURVEY.md 8d): the BASELINE.json configurations as
tensors.  Used by bench.py, __graft_entry__.smoke(), tools/ and the tests -- there is no dataset
and no checkpoint in this tier, so the workload generators are part of the package.

  sca_like_inputs    configs[1]: MSDA operands at the SpatialCrossAttention shape
  dvr_inputs_lidar   configs[2]: sigma volume + LiDAR-like rays
  camera_rig         cfg4: a nuScenes-like 6-camera rig (lidar2img matrices) for point_sampling
"""
import math

import numpy as np
import torch

SCA_LEVELS = ((116, 200), (58, 100), (29, 50), (15, 25))   # 928x1600 input, strides 8..64
IMG_HW = (928, 1600)


def level_tensors(levels, device="cpu"):
    shapes = torch.tensor(levels, dtype=torch.int64, device=device)
    hw = shapes[:, 0] * shapes[:, 1]
    lsi = torch.cat([hw.new_zeros(1), hw.cumsum(0)[:-1]])
    return shapes, lsi


def sca_like_inputs(device, cams=6, Q=40000, seed=0, levels=SCA_LEVELS, heads=8, head_dim=32, points=8,
                    rows=None):
    """Every camera sees a fan of Q pillars of its own frustum: perspective projection of a
    sqrt(Q) x sqrt(Q) polar BEV patch with 4 Z-anchors (-4,-2,0,2 m, camera at 1.5 m), f = 1266 px
    on a 1600x928 image, plus N(0, 4 px) learned-offset noise per (head, level, point)
    (SURVEY.md 8d cfg2).  Bottom anchors of near pillars fall outside the image, as in the real rig.
    `rows`: keep only the first `rows` queries of every camera (the "rebatched" mode, 10240)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    L, P, H = len(levels), points, heads
    K = sum(h * w for h, w in levels)
    n = int(math.isqrt(Q))
    assert n * n == Q
    iy, ix = torch.meshgrid(torch.arange(n), torch.arange(n), indexing="ij")
    depth = 2.0 + 49.0 * (iy.reshape(-1).float() + 0.5) / n               # 2 .. 51 m
    ang = ((ix.reshape(-1).float() + 0.5) / n - 0.5) * math.radians(60.0)
    u = 0.5 + torch.tan(ang) * 1266.0 / 1600.0
    zs = torch.tensor([-4.0, -2.0, 0.0, 2.0])
    v = (491.0 + 1266.0 * (1.5 - zs)[None, :] / depth[:, None]) / 928.0    # [Q, 4]
    ref = torch.stack([u[:, None].expand(-1, 4), v], -1)                   # [Q, 4(z), 2]
    ref = ref[None].expand(cams, -1, -1, -1).clone()
    ref += 0.01 * torch.randn(cams, 1, 1, 2, generator=g)                  # per-camera jitter
    if rows is not None:
        # rebatched mode: a camera keeps an evenly strided subset of its pillars
        keep = torch.linspace(0, Q - 1, rows).round().long()
        ref, Q = ref[:, keep].contiguous(), rows
    ref = ref.to(device)
    wh = torch.tensor([[w, h] for h, w in levels], dtype=torch.float32, device=device)
    dg = torch.Generator(device=device).manual_seed(seed + 1)
    off = 4.0 * torch.randn(cams, Q, H, L, P, 2, device=device, generator=dg) / wh.view(1, 1, 1, L, 1, 2)
    # point p = j*4 + z uses Z-anchor z (spatial_cross_attention.py:356-371)
    loc = off.view(cams, Q, H, L, P // 4, 4, 2) + ref.view(cams, Q, 1, 1, 1, 4, 2)
    loc = loc.view(cams, Q, H, L, P, 2).contiguous()
    attn = torch.softmax(torch.randn(cams, Q, H, L * P, device=device, generator=dg), -1)
    attn = attn.view(cams, Q, H, L, P).contiguous()
    value = torch.randn(cams, K, H, head_dim, device=device, generator=dg)
    grad_out = torch.randn(cams, Q, H * head_dim, device=device, generator=dg)
    shapes, lsi = level_tensors(levels, device)
    return dict(value=value, shapes=shapes, lsi=lsi, loc=loc, attn=attn, grad_out=grad_out)


def dvr_inputs_lidar(M=30000, T=3, grid=(16, 200, 200), seed=0, N=1, pad=0):
    """BASELINE.json configs[2]: sigma [N,T,16,200,200] = softplus(N(0,1)), origin ~ grid centre,
    32-beam LiDAR-like endpoints, range U(2,70) m at 0.512 m/voxel (SURVEY.md 8d cfg3)."""
    rng = np.random.default_rng(seed)
    Z, Y, X = grid
    sigma = np.log1p(np.exp(rng.standard_normal((N, T, Z, Y, X)))).astype(np.float32)
    origin = (np.array([X / 2, Y / 2, Z * 5.0 / 8.0]) + rng.normal(0, 0.5, (N, T, 3))).astype(np.float32)
    beams = np.deg2rad(np.linspace(-30, 10, 32))
    elev = beams[rng.integers(0, 32, (N, M))]
    azim = rng.uniform(-np.pi, np.pi, (N, M))
    rng_m = rng.uniform(2, 70, (N, M)) / 0.512
    tindex = (np.arange(M) * T // M).astype(np.float32)[None].repeat(N, 0)
    d = np.stack([np.cos(elev) * np.cos(azim), np.cos(elev) * np.sin(azim),
                  np.sin(elev) * (Z / 8.0) / (X / 102.4)], -1)  # z voxels are 0.5 m, x/y 0.512 m
    o_per_ray = np.take_along_axis(origin, tindex.astype(np.int64)[..., None].repeat(3, -1), 1)
    points = (o_per_ray + d * rng_m[..., None]).astype(np.float32)
    if pad:
        points[:, -pad:] = np.nan
        tindex[:, -pad:] = -1
    return sigma, origin, points, tindex


def camera_rig(cams=6, img_hw=(900, 1600), f=1266.0, pp=(816.0, 491.0), cam_height=1.5, seed=0):
    """lidar2img [cams,4,4] (float32) of a nuScenes-like rig (SURVEY.md 8d cfg4): yaw
    {0, +-55, +-110, 180} deg, focal 1266 px, principal point (816, 491), cameras 1.5 m above the
    LiDAR origin plane and ~1 m out from the centre, so each BEV pillar projects into 1-2 cameras."""
    yaws = np.deg2rad([0.0, 55.0, -55.0, 110.0, -110.0, 180.0])[:cams]
    rng = np.random.default_rng(seed)
    K = np.array([[f, 0, pp[0], 0], [0, f, pp[1], 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)
    # camera axes in the LiDAR frame: z forward, x right, y down
    mats = []
    for yaw in yaws:
        yaw = yaw + rng.normal(0, 0.01)
        fwd = np.array([np.cos(yaw), np.sin(yaw), 0.0])
        right = np.array([np.sin(yaw), -np.cos(yaw), 0.0])
        down = np.array([0.0, 0.0, -1.0])
        R = np.stack([right, down, fwd], 0)                 # rows: camera axes
        pos = fwd * 1.0 + np.array([0, 0, cam_height])
        E = np.eye(4)
        E[:3, :3] = R
        E[:3, 3] = -R @ pos
        mats.append(K @ E)
    return torch.from_numpy(np.stack(mats, 0).astype(np.float32))


def camera_rig_split(cams=6, f=1266.0, pp=(816.0, 491.0), cam_height=1.5, seed=0, yaws_deg=None):
    """(cam2img, lidar2cam), each [cams, 4, 4] float64, of camera_rig's rig: the intrinsics and the extrinsics that
    the reference's image pipeline keeps apart (CropResizeFlipImage rescales cam2img, then forms
    lidar2img = cam2img @ lidar2cam).  Their product is camera_rig(cams) before its float32 cast.  `yaws_deg`: the
    cameras' yaws (default nuScenes-like six)."""
    yaws = np.deg2rad([0.0, 55.0, -55.0, 110.0, -110.0, 180.0] if yaws_deg is None else yaws_deg)[:cams]
    rng = np.random.default_rng(seed)
    K = np.array([[f, 0, pp[0], 0], [0, f, pp[1], 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)
    exts = []
    for yaw in yaws:
        yaw = yaw + rng.normal(0, 0.01)
        fwd = np.array([np.cos(yaw), np.sin(yaw), 0.0])
        right = np.array([np.sin(yaw), -np.cos(yaw), 0.0])
        R = np.stack([right, np.array([0.0, 0.0, -1.0]), fwd], 0)
        E = np.eye(4)
        E[:3, :3] = R
        E[:3, 3] = -R @ (fwd * 1.0 + np.array([0, 0, cam_height]))
        exts.append(E)
    return np.stack([K] * len(exts), 0), np.stack(exts, 0)


def lidar_cloud(rng, n, lattice=64):
    """A LiDAR-like float32 [n, 5] cloud (x, y, z, intensity, ring) on a 1/lattice m grid: 32 rings of ground and
    walls, a few percent of the points inside the ego box (-0.8..0.8, -1.5..2.5), inside the 1 m square around the
    sensor and outside the +-51.2 m range."""
    kind = rng.choice(4, n, p=[0.9, 0.04, 0.03, 0.03])
    ring = rng.integers(0, 32, n)
    ang = rng.uniform(-np.pi, np.pi, n)
    r = np.where(ring < 24, 2.5 + 1.6 * ring + rng.normal(0, 0.05, n), rng.uniform(5.0, 45.0, n))
    z = np.where(ring < 24, -1.8 + rng.normal(0, 0.03, n), rng.uniform(-1.5, 2.5, n))
    x, y = r * np.cos(ang), r * np.sin(ang)
    ego, close = kind == 1, kind == 2
    x[ego], y[ego] = rng.uniform(-0.8, 0.8, ego.sum()), rng.uniform(-1.5, 2.5, ego.sum())
    x[close], y[close] = rng.uniform(-1.0, 1.0, close.sum()), rng.uniform(-1.0, 1.0, close.sum())
    far = kind == 3
    x[far], y[far] = 51.2 + rng.uniform(0.0, 20.0, far.sum()) * np.sign(x[far]), y[far] * 1.5
    pts = np.stack([x, y, z, rng.integers(0, 100, n), ring], 1)
    return (np.round(pts * lattice) / lattice).astype(np.float32)


def camera_image(rng, hw):
    """A camera-like uint8 [h, w, 3] BGR image: a smooth random field (a 1/32-scale random image, bicubic-upsampled)
    with a little per-pixel noise, so that it compresses like a photograph rather than like white noise."""
    import cv2
    h, w = hw
    small = rng.integers(0, 256, (h // 32 + 2, w // 32 + 2, 3), dtype=np.uint8)
    img = cv2.resize(small, (w, h), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    img += rng.integers(-4, 5, img.shape, dtype=np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


def sweep_pose(rng, k):
    """(sensor2lidar_rotation, sensor2lidar_translation) float64 of the k-th earlier sweep: the ego moving about
    0.5 m and turning about 0.3 degrees per sweep, with a slight roll."""
    yaw, roll = rng.normal(0, 0.005) * k, rng.normal(0, 0.001)
    cz, sz, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(roll), np.sin(roll)
    R = np.array([[cz, -sz, 0.0], [sz, cz, 0.0], [0.0, 0.0, 1.0]]) @ np.array([[1.0, 0, 0], [0, cr, -sr], [0, sr, cr]])
    t = np.array([-0.5 * k + rng.normal(0, 0.02), rng.normal(0, 0.02), rng.normal(0, 0.01)])
    return R, t


LIDAR2EGO_TRANSLATION = [0.943713, 0.0, 1.84023]                          # nuScenes' roof LiDAR mounting
LIDAR2EGO_ROTATION = [0.7077955119163518, -0.006492242056004365, 0.010646214713995808, -0.7063073142877817]


def drive(frames, seed=0, scene_change=None, dt=0.5):
    """A seeded nuScenes-like drive of `frames` keyframes `dt` s apart -> one pose dict per frame (the dataset's info
    fields): ego2global_translation / rotation (w, x, y, z), lidar2ego_translation / rotation, an 18-value can_bus
    (position, orientation, acceleration, rotation rate, velocity, two zeros, as nuScenes' CAN bus pose message) and
    scene_token.  Speed up to about 15 m/s and yaw rate within +-10 deg/s, with small pitch / roll.
    `scene_change` = i: frames i .. end belong to another scene, starting elsewhere on the map."""
    rng = np.random.default_rng(seed + 7919)
    out = []
    pos, yaw, scene = rng.uniform(300, 1500, 3) * np.array([1, 1, 0]), rng.uniform(-np.pi, np.pi), 0
    speed = rng.uniform(0, 15)
    for t in range(frames):
        if scene_change is not None and t == scene_change:
            pos, yaw, scene = rng.uniform(300, 1500, 3) * np.array([1, 1, 0]), rng.uniform(-np.pi, np.pi), 1
            speed = rng.uniform(0, 15)
        elif t > 0:
            rate = np.deg2rad(rng.uniform(-10, 10))
            accel = rng.uniform(-2, 2)
            speed = float(np.clip(speed + accel * dt, 0, 15))
            yaw += rate * dt
            pos = pos + speed * dt * np.array([np.cos(yaw), np.sin(yaw), 0.0])
        pitch, roll = rng.normal(0, 0.01), rng.normal(0, 0.005)
        cy, sy, cp, sp, cr, sr = (np.cos(yaw / 2), np.sin(yaw / 2), np.cos(pitch / 2), np.sin(pitch / 2),
                                  np.cos(roll / 2), np.sin(roll / 2))
        q = [cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy,
             cr * cp * sy - sr * sp * cy]
        can_bus = np.concatenate([pos, q, rng.normal(0, 0.5, 3), rng.normal(0, 0.05, 3), [speed, 0.0, 0.0],
                                  [0.0, 0.0]])
        out.append(dict(ego2global_translation=[float(v) for v in pos], ego2global_rotation=[float(v) for v in q],
                        lidar2ego_translation=list(LIDAR2EGO_TRANSLATION), lidar2ego_rotation=list(LIDAR2EGO_ROTATION),
                        can_bus=can_bus, scene_token=f"synthetic-{seed}-{scene}"))
    return out


NUPLAN_YAWS = (0.0, 45.0, -45.0, 90.0, -90.0, 135.0, -135.0, 180.0)
NUPLAN_IMG_HW = (1080, 1920)


def nuplan_camera_rig_split():
    """(cam2img, lidar2cam) of an 8-camera 1920 x 1080 rig like OpenScene's."""
    return camera_rig_split(8, f=1545.0, pp=(960.0, 560.0), yaws_deg=NUPLAN_YAWS)


def write_pcd(path, cloud, garbage=16):
    """Writes float32 [n, 6] (x, y, z, intensity, ring, lidar_info) as a binary .pcd with nuPlan's six fields: the
    coordinates and intensity float32, ring uint16 and lidar_info uint8 (the values are cast), followed by `garbage`
    zero bytes, as nuPlan's files carry trailing bytes."""
    row = np.dtype([("x", np.float32), ("y", np.float32), ("z", np.float32), ("intensity", np.float32),
                    ("ring", np.uint16), ("lidar_info", np.uint8)])
    rec = np.zeros(len(cloud), row)
    for j, name in enumerate(row.names):
        rec[name] = cloud[:, j]
    head = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity ring lidar_info\n"
            "SIZE 4 4 4 4 2 1\nTYPE F F F F U U\nCOUNT 1 1 1 1 1 1\n"
            f"WIDTH {len(cloud)}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {len(cloud)}\nDATA binary\n")
    with open(path, "wb") as fh:
        fh.write(head.encode("utf8") + rec.tobytes() + bytes(garbage))


def nuplan_cloud(rng, n):
    """lidar_cloud's points with nuPlan's six columns: the ring as column 4 and a lidar_info id in 0..4."""
    c = lidar_cloud(rng, n)
    return np.concatenate([c, rng.integers(0, 5, (n, 1)).astype(np.float32)], 1)
