"""Shared inputs of the point pipeline tests: the golden cases of tests/golden/point_pipeline.npz (written by
tools/make_golden_point_pipeline.py from the reference's own statements) replayed through
vidar_b200.point_pipeline's transforms."""
import json
import os

import numpy as np

from vidar_b200 import point_pipeline as pp

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "point_pipeline.npz")


def golden():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["cases"]))


def transforms(meta):
    sweeps = dict(meta["sweeps_kwargs"])
    sampler = dict(meta["sampler_kwargs"])
    return [pp.LoadPointsFromFile(coord_type="LIDAR", load_dim=5, use_dim=5),
            pp.CustomLoadPointsFromMultiSweeps(**sweeps), pp.CustomVoxelBasedPointSampler(**sampler)]


def frame_info(z, name, f, root):
    """The dataset's results dict of frame f, its files written under root."""
    def put(key):
        path = os.path.join(root, key + ".bin")
        if not os.path.exists(path):
            z[key].tofile(path)
        return path
    pose, sts = z[f"{name}.{f}.pose"], z[f"{name}.{f}.sweep_ts"]
    sweeps = [dict(data_path=put(f"{name}.{f}.sweep{j}"), timestamp=int(sts[j]),
                   sensor2lidar_rotation=pose[j, :9].reshape(3, 3).copy(), sensor2lidar_translation=pose[j, 9:].copy())
              for j in range(len(sts))]
    return dict(pts_filename=put(f"{name}.{f}.key"), timestamp=int(z[f"{name}.{f}.ts"]) / 1e6, sweeps=sweeps)


def run_order(meta):
    """(frame, gathered) in the dataset's order: previous frames, the current frame's draw-only run, then the
    current and future frames."""
    p, n = meta["current"], len(meta["frames"])
    return [(f, True) for f in range(p)] + [(p, False)] + [(f, True) for f in range(p, n)]


def state_row():
    st = np.random.get_state()
    return np.concatenate([st[1].astype(np.int64), [st[2], st[3]]]), np.float64(st[4])


def replay(z, meta, root):
    """Run the case's frames through the package's transforms after the golden's seeding -> (the gathered frames'
    results in queue order, [(MT key + pos + has_gauss, cached gaussian)] after every call)."""
    steps = transforms(meta)
    np.random.seed(meta["seed"])
    states, gathered = [], []
    for f, keep in run_order(meta):
        results = frame_info(z, meta["name"], f, root)
        for s in steps:
            results = s(results)
            states.append(state_row())
        if keep:
            gathered.append(results)
    return gathered, states
