"""Pre-training samples from their files: the host half of every pipeline in DataLoader workers, the device half
prefetched on a side stream while the previous step runs.

`SampleLoader(model, samples, num_workers, prefetch)` takes one queue of results dicts per sample, as a dataset's
get_data_info hands them to its pipeline (`pretrain.synthetic_sample(..., files=True)` makes one).  Per sample, a
worker (`QueueDataset`) runs, in the order `SyntheticViDAR.forward_train` runs the same transforms:

  * the train point transforms of the GT frames, in queue order (`run_point_transforms`: file reads, sweep
    selection, the voxel sampler's shuffles; the host half of `gt_points_of`);
  * for the image frames, oldest first: `jpeg.LoadMultiViewImageFromFiles` (file reads and marker parsing, no
    draws), then the image transforms' draws (`run_image_transforms`, with `aug_param` carried across frames; the
    host half of `frame_transforms`).

With `test_mode=True` a worker runs the config's test pipeline instead: LoadPointsFromFile on the GT frames, and
LoadMultiViewImageFromFiles, normalisation and padding on the image frames, with no draw at all.

It returns the parsed JPEG records, the image plans and the point plans, not pixels.  The model's own draws (A1 / A2
and the supervised future frame, `host_draws`) and GridMask's stay in the training process, as the reference's
detector makes them there.  Workers are seeded as mmdet's `worker_init_fn` seeds them: numpy, `random` and torch with
seed + rank * num_workers + worker_id, so a run is reproducible for a fixed seed and worker count.  With
num_workers=0 the dataset draws from the training process's generators when a sample is fetched -- with
prefetch > 0, one sample ahead of the step.

The device half of a sample, on the training process: one packed upload and `jpeg.decode_frames` of this rank's
backbone cameras (`model.backbone_cams()`), `image_aug.apply_multiview` of each frame, and `gather_gt_points`.  With
`prefetch` = k > 0 it runs on a side stream k samples ahead: the side stream first waits on the step's stream (so it
never reads a buffer the step is still writing), and when the sample is handed out the step's stream waits on an
event recorded after its work.  The side stream's wait at each launch also orders the reuse of a dropped sample's
blocks (they belong to the side stream's pool) after every step queued before that launch; each tensor the step
reads is in addition `record_stream`-ed on the step's stream, so that it is not reused before the step is done with
it however long the caller keeps the sample.  No host sync.  With prefetch=0 the same work
runs on the current stream when the sample is handed out, just before the step: the reference's order.
"""
import collections
import copy
import functools
import random

import numpy as np
import torch

from . import ego_motion, image_aug, jpeg


def run_image_transforms(transforms, frames):
    """The image transforms over the results dicts of a queue's image frames, oldest first; the first frame's
    `aug_param` (crop / resize / flip) is carried to the later ones -> the frames' results."""
    out, aug_param = [], None
    for results in frames:
        if aug_param is not None:
            results["aug_param"] = copy.deepcopy(aug_param)
        for transform in transforms:
            results = transform(results)
        aug_param = copy.deepcopy(results.get("aug_param"))
        out.append(results)
    return out


def run_point_transforms(transforms, infos):
    """The point transforms over the results dicts of a queue's GT frames, in queue order -> their results."""
    frames = []
    for info in infos:
        results = dict(info)
        for step in transforms:
            results = step(results)
        frames.append(results)
    return frames


class QueueDataset(torch.utils.data.Dataset):
    """The host half of a sample: `samples[i]` is a queue of results dicts; frames with `img_filename` are the image
    frames, frames with `pts_filename` the GT frames.  -> dict(frames=[image results], points=[point results],
    index=i).  Makes no CUDA call.  `test_mode`: an image frame brings its `lidar2img` (the test chain does not form
    it) instead of `cam2img` and `lidar2cam`.  `poses`: every frame brings its pose fields, and the result also holds
    poses=[metas per image frame] (`ego_motion.queue_metas`).  `lidar2img`: whether an image frame brings the
    dataset's `lidar2img` (default: in test mode), as the OpenScene train chain needs it too -- it has no crop step
    to form it."""

    def __init__(self, samples, image_transforms, point_transforms, test_mode=False, poses=False, lidar2img=None):
        self.samples = list(samples)
        self.poses = bool(poses)
        self.image_transforms = list(image_transforms)
        self.point_transforms = list(point_transforms)
        self.test_mode = bool(test_mode)
        self.lidar2img = self.test_mode if lidar2img is None else bool(lidar2img)
        self.load_images = jpeg.LoadMultiViewImageFromFiles(to_float32=True)

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, index):
        queue = self.samples[index]
        points = run_point_transforms(self.point_transforms, [f for f in queue if "pts_filename" in f])
        keys = ("lidar2img",) if self.lidar2img else ("cam2img", "lidar2cam")
        frames = []
        for f in queue:
            if "img_filename" in f:
                if self.lidar2img and "lidar2img" not in f:
                    raise ValueError(f"sample {index}: an image frame of this pipeline needs its lidar2img")
                frames.append(self.load_images(dict(img_filename=list(f["img_filename"]),
                                                    **{k: [np.array(m, np.float64) for m in f[k]] for k in keys})))
        if not frames or not points:
            raise ValueError(f"sample {index}: a queue needs image frames (img_filename) and GT frames (pts_filename)")
        poses = ego_motion.queue_metas(queue) if self.poses else None
        return dict(frames=run_image_transforms(self.image_transforms, frames), points=points, index=index,
                    poses=poses)


def seed_worker(worker_id, num_workers, rank, seed):
    """mmdet's worker_init_fn: numpy, `random` and torch seeded with seed + rank * num_workers + worker_id."""
    worker_seed = num_workers * rank + worker_id + seed
    np.random.seed(worker_seed)
    random.seed(worker_seed)
    torch.manual_seed(worker_seed)


def _one(sample):
    return sample


class SampleLoader:
    """Iterates over `samples` (queues of results dicts), yielding samples for `pretrain.train_step` /
    `SyntheticViDAR.forward_train`: dict(img=[float32 [len(cams), 3, Hp, Wp] per image frame: the decoded and
    pipelined images of this rank's backbone cameras], img_metas=[[dict(lidar2img, img_shape)] per image frame],
    gt_points=[1, R, 5] on the device, lidar2img=None, index).

    `model`: a `SyntheticViDAR` built with image_pipeline=True and point_pipeline=True, whose train transforms the
    workers run (`model.image_transforms`, `model.point_transforms[0]`).
    `test_mode=True` runs the config's test pipeline instead, as its val / test datasets do: per image frame
    `LoadMultiViewImageFromFiles`, normalisation and padding (`image_aug.config_test_pipeline`: no draw, no crop or
    resize), with each frame's `lidar2img` taken from its results dict as it is; per GT frame LoadPointsFromFile only
    (`model.point_transforms[1]`).  The model then needs point_pipeline=True only, and each frame's img_metas also
    carry `filename`, its camera files, as the reference's metas do (`pretrain.evaluate` keys its feature reuse on
    them).  The device half is the same.
    `num_workers`: DataLoader worker processes (0: the host half on this process).  `prefetch`: samples whose device
    half runs ahead on a side stream (0: on the current stream, at hand-out).  `seed` and `rank` seed the workers;
    `rank` is the data-parallel replica (`grid.replica`): every rank of a shard group passes the same value and
    iterates the same samples, so their draws agree, and each decodes only its own backbone cameras.
    A model built with openscene=True runs the OpenScene chains (`model.image_transforms`,
    `model.test_image_transforms`, the nuPlan point loaders), and its image frames bring their `lidar2img` in both
    modes.  `ego_mask`: union2one's ego box for gt_points (default the configs' `pretrain.EGO_MASK`; the submit
    config's is (0, 0, 0, 0)).
    A model built with ego_motion=True needs every queue frame's pose fields (`ego_motion.POSE_KEYS`); the workers
    then run `ego_motion.queue_metas` on the queue and each image frame's img_metas carry its result."""

    def __init__(self, model, samples, num_workers=0, prefetch=1, seed=0, rank=0, test_mode=False, ego_mask=None):
        if test_mode and model.point_transforms is None:
            raise ValueError("SampleLoader(test_mode=True): the model must be built with point_pipeline=True")
        if not test_mode and (model.image_transforms is None or model.point_transforms is None):
            raise ValueError("SampleLoader: the model must be built with image_pipeline=True and point_pipeline=True")
        if num_workers < 0 or prefetch < 0:
            raise ValueError(f"SampleLoader: num_workers and prefetch must be >= 0 (got {num_workers}, {prefetch})")
        self.model, self.prefetch, self.num_workers = model, int(prefetch), int(num_workers)
        self.test_mode = bool(test_mode)
        self.ego_mask = ego_mask
        lidar2img = True if getattr(model, "openscene", False) else None
        if test_mode:
            self.dataset = QueueDataset(samples, model.test_image_transforms, model.point_transforms[1], True,
                                        poses=getattr(model, "ego_motion", False), lidar2img=lidar2img)
        else:
            self.dataset = QueueDataset(samples, model.image_transforms, model.point_transforms[0],
                                        poses=getattr(model, "ego_motion", False), lidar2img=lidar2img)
        init = functools.partial(seed_worker, num_workers=num_workers, rank=rank, seed=seed) if num_workers else None
        self.host_loader = torch.utils.data.DataLoader(self.dataset, batch_size=None, shuffle=False,
                                                       num_workers=num_workers, collate_fn=_one, worker_init_fn=init)
        self.stream = None

    def __len__(self):
        return len(self.dataset)

    def device_sample(self, host):
        """The device half of one host sample, on the current stream."""
        model = self.model
        dev = model.bev_embedding.weight.device
        cams = model.backbone_cams()
        frames = host["frames"]
        if cams:
            decoded = jpeg.decode_frames(frames, dev, cams=cams)
            img = [image_aug.apply_multiview(raw, r, cams) for r, raw in zip(frames, decoded)]
        else:
            img = [torch.empty((0, 3, *r["img_aug"].pad_hw), dtype=torch.float32, device=dev) for r in frames]
        poses = host.get("poses") or [{}] * len(frames)
        metas = [[dict(lidar2img=np.stack(r["lidar2img"]), img_shape=r["img_shape"],
                       **(dict(filename=list(r["filename"])) if self.test_mode else {}), **p)]
                 for r, p in zip(frames, poses)]
        gt_points = model.gather_points(host["points"], *(() if self.ego_mask is None else (self.ego_mask,)))
        return dict(img=img, img_metas=metas, gt_points=gt_points, lidar2img=None,
                    index=host["index"])

    def __iter__(self):
        it = iter(self.host_loader)
        if self.prefetch == 0:
            for host in it:
                yield self.device_sample(host)
            return
        dev = self.model.bev_embedding.weight.device
        if self.stream is None:
            self.stream = torch.cuda.Stream(dev)
        pending = collections.deque()

        def launch():
            host = next(it, None)
            if host is None:
                return
            self.stream.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(self.stream):
                sample = self.device_sample(host)
                done = torch.cuda.Event()
                done.record(self.stream)
            pending.append((sample, done))

        for _ in range(self.prefetch):
            launch()
        while pending:
            sample, done = pending.popleft()
            step = torch.cuda.current_stream(dev)
            step.wait_event(done)
            for t in [*sample["img"], sample["gt_points"]]:
                if t.numel():
                    t.record_stream(step)
            launch()                                  # the next sample's device half overlaps this step
            yield sample
