"""Device-resident image sets: the input of a captured training or test step made on the GPU.

The reference feeds every step from a DataLoader whose workers decode an image, resize it, jitter its colours
(clustered sets), normalise it and load its ground truth; the loop then shifts the image (util.random_shift) and copies
everything to the device.  Here the decode and the resize run once, when the set is built, and the set keeps its uint8
images, ground truth and attachments in device memory (or in mapped pinned host memory).  Each step's tensors are then made
by five kernels (esacb200_data_step_async) that a CUDA graph captures with the step, so a training loop is

    for g in plan.groups:
        dataset.step(g)          # captured in graphs[g]
        graphs[g].replay()

The randomness stays the reference's: `make_plan` makes the reference loop's random calls (the dataset's `random.choice` /
`randint` or `img_sampler.sample()`, ColorJitter.get_params, the shuffling sampler's permutation, util.random_shift's two
`randint`) in the reference's order, by iterating a DataLoader(num_workers=0) over an index-only dataset.  It runs once per
epoch and is uploaded with one copy (DeviceImageSet.load_plan); the device does only the pixel work, bitwise what PIL and
torchvision compute on the host.
"""
from __future__ import annotations

import math
import os
import random
from dataclasses import dataclass

import numpy as np

from . import api

ROOM_MEAN, ROOM_STD = 0.4, 0.25           # room_dataset.py:91-99, statistics of the 7-Scenes training set
CLUSTER_MEAN, CLUSTER_STD = 0.3639, 0.2074  # cluster_dataset.py:182-200, statistics of the Aachen day training set
MAX_SHIFT = 4                             # util.random_shift's bound, int(Expert.OUTPUT_SUBSAMPLE / 2)
OPS = {"brightness": api.DATA_BRIGHTNESS, "contrast": api.DATA_CONTRAST, "saturation": api.DATA_SATURATION}


def _three(v, what: str) -> tuple:
    a = np.asarray(v, np.float64).reshape(-1)
    if a.shape == (1,):
        a = np.repeat(a, 3)
    if a.shape != (3,) or not np.isfinite(a).all():
        raise ValueError(f"{what} must be a number or three finite numbers, got {v!r}")
    return tuple(float(x) for x in a)


def rgb_image(image) -> np.ndarray:
    """A decoded image as contiguous uint8 [H,W,3]: a gray [H,W] image copied into three channels (color.gray2rgb,
    room_dataset.py:156-157)."""
    a = image.numpy() if type(image).__module__.startswith("torch") else np.asarray(image)
    if a.dtype != np.uint8:
        raise ValueError(f"images must be uint8, got {a.dtype}")
    if a.ndim == 2:
        a = np.stack([a, a, a], axis=-1)
    if a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
        raise ValueError(f"images must be [H,W,3] RGB or [H,W] gray, got {list(a.shape)}")
    if max(a.shape[:2]) > api.DATA_MAX_SIDE:
        raise ValueError(f"image {a.shape[0]}x{a.shape[1]} has a side above {api.DATA_MAX_SIDE}")
    return np.ascontiguousarray(a)


@dataclass
class Plan:
    """One epoch of steps: rows (api.DATA_ROW, B per step, in step order), groups (the shape group of each step) and B."""
    rows: np.ndarray
    groups: list
    batch: int


class DeviceImageSet:
    """A set of decoded, resized uint8 RGB images with their poses, cameras, scenes, optional ground truth and optional
    attachments, held on the device (storage="device") or in mapped pinned host memory (storage="pinned").

    images: N uint8 [H,W,3] (or gray [H,W]) arrays or tensors, already resized; poses: [N,4,4] camera->world, stored as
    float32 (offsets already applied); focal: N focal lengths already scaled by imsize / min(h, w) (float64; the camera
    holds their float32 rounding); scenes: N ints (-1 for a clustered set); gt: None or N float32 [3,h,w] maps;
    attachments: name -> float32 tensor [N, ...] (a gating-target row, a stand-in prior...); mean / std: the
    normalisation (one number or three); plan_capacity: the most rows a plan may hold (default max(N, 1000): the
    reference's room epoch is 1000 items).  The images are grouped by (image shape, ground-truth shape), in order of first
    appearance: `groups` lists the shapes, `group_of` the group of each image."""

    def __init__(self, images, poses, focal, scenes, gt=None, attachments=None, mean=ROOM_MEAN, std=ROOM_STD,
                 storage: str = "device", plan_capacity: int | None = None, device: int | None = None):
        import torch
        if storage not in ("device", "pinned"):
            raise ValueError(f"storage must be 'device' or 'pinned', got {storage!r}")
        imgs = [rgb_image(im) for im in images]
        N = len(imgs)
        if N < 1:
            raise ValueError("a set needs at least one image")
        poses = torch.as_tensor(np.asarray(poses)).float()
        if tuple(poses.shape) != (N, 4, 4):
            raise ValueError(f"poses must be [{N},4,4], got {list(poses.shape)}")
        focal = np.asarray(focal, np.float64).reshape(-1)
        scenes = np.asarray(scenes, np.int64).reshape(-1)
        if focal.shape != (N,) or scenes.shape != (N,):
            raise ValueError(f"focal and scenes must hold {N} values each, got {focal.shape[0]} and {scenes.shape[0]}")
        if gt is not None:
            gt = [torch.as_tensor(g) for g in gt]
            if len(gt) != N:
                raise ValueError(f"gt must hold {N} maps, got {len(gt)}")
            for i, g in enumerate(gt):
                if g.dtype != torch.float32 or g.dim() != 3 or g.shape[0] != 3 or min(g.shape) < 1:
                    raise ValueError(f"gt[{i}] must be a float32 [3,h,w] map, got {g.dtype} {list(g.shape)}")
        attachments = dict(attachments or {})
        if len(attachments) > api.DATA_MAX_ATTACH:
            raise ValueError(f"at most {api.DATA_MAX_ATTACH} attachments, got {len(attachments)}")
        for name, a in attachments.items():
            if not isinstance(a, torch.Tensor) or a.dtype != torch.float32 or a.dim() < 1 or a.shape[0] != N or a.numel() == 0:
                raise ValueError(f"attachment {name!r} must be a float32 tensor [{N}, ...] with elements")
            if name in ("image", "shifts", "cameras", "gt_poses", "gt_coords", "scenes", "indices", "status"):
                raise ValueError(f"attachment name {name!r} is taken by an output")
        self.mean, self.std = _three(mean, "mean"), _three(std, "std")
        if 0.0 in self.std:
            raise ValueError("std must be nonzero")
        capacity = max(N, 1000) if plan_capacity is None else int(plan_capacity)
        if capacity < 1:
            raise ValueError(f"plan_capacity must be positive, got {capacity}")
        if not torch.cuda.is_available():
            raise RuntimeError("DeviceImageSet needs a CUDA device; there is no CPU path")

        self.N, self.storage, self.capacity = N, storage, capacity
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else int(device))
        shapes = [(im.shape[0], im.shape[1]) + ((int(gt[i].shape[1]), int(gt[i].shape[2])) if gt is not None else (0, 0))
                  for i, im in enumerate(imgs)]
        self.groups = list(dict.fromkeys(shapes))
        index = {s: g for g, s in enumerate(self.groups)}
        self.group_of = np.array([index[s] for s in shapes], np.int32)

        rec = np.zeros(N, api.DATA_IMAGE)
        sizes = np.array([im.nbytes for im in imgs], np.int64)
        rec["pixels"] = np.concatenate([[0], np.cumsum(sizes)[:-1]])
        rec["gt"] = -1
        if gt is not None:
            gsizes = np.array([g.numel() for g in gt], np.int64)
            rec["gt"] = np.concatenate([[0], np.cumsum(gsizes)[:-1]])
        rec["focal"], rec["scene"] = focal, scenes
        rec["pose"] = poses.reshape(N, 16).numpy()
        rec["group"] = self.group_of
        rec["H"], rec["W"] = [s[0] for s in shapes], [s[1] for s in shapes]
        rec["gt_h"], rec["gt_w"] = [s[2] for s in shapes], [s[3] for s in shapes]
        self.records = rec

        def keep(t):
            return t.to(self.device) if storage == "device" else t.pin_memory()

        self.pixels = keep(torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])))
        self.gt = keep(torch.cat([g.reshape(-1) for g in gt])) if gt is not None else None
        self.attachments = {name: keep(a.contiguous()) for name, a in attachments.items()}
        self.images = torch.from_numpy(rec.view(np.uint8).reshape(N, api.DATA_IMAGE.itemsize)).to(self.device)
        self.plan_rows = torch.zeros((capacity, api.DATA_ROW.itemsize // 4), dtype=torch.int32, device=self.device)
        self.state = torch.zeros(api.DATA_STATE, dtype=torch.int64, device=self.device)
        self._outputs = {}

    def __len__(self):
        return self.N

    def outputs(self, group: int, B: int = 1) -> dict:
        """The static tensors step(group, B) writes, made once per (group, B): image float32 [B,3,H,W], shifts int32 [B,2],
        cameras float32 [B,3] (f, W/2, H/2), gt_poses float32 [B,4,4], gt_coords float32 [B,3,h,w] (sets with ground
        truth), scenes and indices int64 [B], one float32 [B, ...] tensor per attachment, and status int32 [1] (0 ok,
        1 the plan is exhausted, 2 a row of another group; on 1 and 2 nothing else is written)."""
        import torch
        key = self._key(group, B)
        if key not in self._outputs:
            H, W, h, w = self.groups[key[0]]
            dev = self.device
            out = {"image": torch.zeros((B, 3, H, W), device=dev), "shifts": torch.zeros((B, 2), dtype=torch.int32, device=dev),
                   "cameras": torch.zeros((B, 3), device=dev), "gt_poses": torch.zeros((B, 4, 4), device=dev),
                   "scenes": torch.zeros(B, dtype=torch.int64, device=dev),
                   "indices": torch.zeros(B, dtype=torch.int64, device=dev)}
            if self.gt is not None:
                out["gt_coords"] = torch.zeros((B, 3, h, w), device=dev)
            for name, a in self.attachments.items():
                out[name] = torch.zeros((B,) + tuple(a.shape[1:]), device=dev)
            out["status"] = torch.zeros(1, dtype=torch.int32, device=dev)
            self._outputs[key] = (out, torch.zeros(B, dtype=torch.int64, device=dev))
        return self._outputs[key][0]

    def _key(self, group, B):
        if isinstance(group, bool) or not isinstance(group, (int, np.integer)) or not 0 <= group < len(self.groups):
            raise ValueError(f"group must be an int in [0, {len(self.groups)}), got {group!r}")
        if isinstance(B, bool) or not isinstance(B, (int, np.integer)) or not 1 <= B <= api.DATA_MAX_BATCH:
            raise ValueError(f"B must be an int in [1, {api.DATA_MAX_BATCH}], got {B!r}")
        return int(group), int(B)

    def step(self, group: int, B: int = 1) -> dict:
        """Enqueues one step of B images of `group` on torch's current stream (capturable: no synchronisation, no
        allocation once outputs(group, B) exists) and returns its outputs."""
        out = self.outputs(group, B)
        work = self._outputs[self._key(group, B)][1]
        names = list(self.attachments)
        api.data_step_async(self.pixels, self.images, self.plan_rows, self.state, int(group), self.mean, self.std, work,
                            out["image"], out["shifts"], out["cameras"], out["gt_poses"], out["scenes"], out["indices"],
                            out["status"], gt=self.gt, outCoords=out.get("gt_coords"),
                            attachments=[self.attachments[n] for n in names], outAttachments=[out[n] for n in names])
        return out

    def load_plan(self, plan: Plan):
        """Uploads the plan's rows and resets the position, ordered on torch's current stream.  Call it outside capture,
        between replays; the plan buffer never moves, so captured steps read the new rows."""
        import torch
        rows = check_plan(plan, self.N, self.group_of, self.capacity)
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("load_plan copies from the host: call it outside capture, between replays")
        n = rows.shape[0]
        host = torch.from_numpy(np.ascontiguousarray(rows).view(np.int32).reshape(n, -1))
        self.plan_rows[:n].copy_(host)
        self.state.copy_(torch.tensor([0, n], dtype=torch.int64))

    def plan(self, draws, batch: int = 1, shuffle: bool = True, shift: bool = True) -> Plan:
        """make_plan over this set's groups."""
        return make_plan(draws, self.group_of, batch=batch, shuffle=shuffle, shift=shift)


def check_plan(plan: Plan, n_images: int, group_of, capacity: int) -> np.ndarray:
    """The rows of a plan a set of n_images images (groups group_of) with room for `capacity` rows can load; raises
    ValueError otherwise."""
    rows = np.asarray(plan.rows)
    if rows.dtype != api.DATA_ROW or rows.ndim != 1:
        raise ValueError(f"plan rows must be a 1-d array of api.DATA_ROW, got {rows.dtype} {rows.shape}")
    n, B = rows.shape[0], int(plan.batch)
    if n > capacity:
        raise ValueError(f"the plan holds {n} rows, more than the set's plan capacity {capacity}")
    if B < 1 or n != B * len(plan.groups):
        raise ValueError(f"the plan holds {n} rows for {len(plan.groups)} steps of {B}")
    img = rows["image"]
    if n and (img.min() < 0 or img.max() >= n_images):
        raise ValueError(f"plan rows name images outside [0, {n_images})")
    if n and (np.abs(rows["padX"]).max() > api.DATA_MAX_SIDE or np.abs(rows["padY"]).max() > api.DATA_MAX_SIDE):
        raise ValueError(f"plan pads outside [-{api.DATA_MAX_SIDE}, {api.DATA_MAX_SIDE}]")
    if n and not np.array_equal(np.asarray(group_of)[img].reshape(-1, B), np.repeat(np.asarray(plan.groups), B).reshape(-1, B)):
        raise ValueError("plan.groups does not hold the shape group of every step's images")
    for r in rows:
        k = int(r["n_ops"])
        ops = [int(o) for o in r["ops"][:k]] if 0 <= k <= 3 else [-1]
        if any(o not in OPS.values() for o in ops) or len(set(ops)) != len(ops) or not np.isfinite(r["factors"][:k]).all():
            raise ValueError(f"plan row {r} has a bad jitter: need n_ops in [0, 3], distinct ops of {OPS} and finite factors")
    return rows


# ------------------------------------------------------------------------------------------------
# the planner: the reference loop's random calls, in its order
# ------------------------------------------------------------------------------------------------
def _jitter_row(jitter):
    """ColorJitter.get_params as the transform calls it (cluster_dataset.py:186-189), as (n_ops, ops[3], factors[3]) in the
    order ColorJitter.forward applies them."""
    if jitter is None:
        return 0, [0, 0, 0], [0.0, 0.0, 0.0]
    fn_idx, b, c, s, _ = jitter.get_params(jitter.brightness, jitter.contrast, jitter.saturation, jitter.hue)
    factors = {api.DATA_BRIGHTNESS: b, api.DATA_CONTRAST: c, api.DATA_SATURATION: s}
    ops = [int(i) for i in fn_idx if int(i) in factors and factors[int(i)] is not None]
    return len(ops), ops + [0] * (3 - len(ops)), [float(factors[o]) for o in ops] + [0.0] * (3 - len(ops))


def _check_jitter(jitter):
    if jitter is not None and jitter.hue is not None:
        raise ValueError("hue jitter is not supported: the reference's datasets jitter brightness, contrast and saturation")


class RoomDraws:
    """The random calls of RoomDataset.__getitem__ (room_dataset.py:105-149) for a set whose scene s holds
    scene_counts[s] images (set images in scene order): a random image of a random scene in training with scene < 0
    (epoch of 1000), image `idx` of `scene` for scene >= 0, image idx of the environment in test.  Items are the set's
    image index and an empty jitter."""

    def __init__(self, scene_counts, scene: int = -1, training: bool = True):
        self.counts = [int(c) for c in scene_counts]
        self.starts = np.concatenate([[0], np.cumsum(self.counts)]).astype(int).tolist()
        self.scene, self.training = int(scene), bool(training)

    def __len__(self):
        if self.scene >= 0:
            return self.counts[self.scene]
        return 1000 if self.training else self.starts[-1]

    def __getitem__(self, idx):
        if self.scene >= 0:
            image = self.starts[self.scene] + idx
        elif self.training:
            s = random.choice(range(len(self.counts)))   # random.choice(self.scenes): the draw depends on the length only
            image = self.starts[s] + random.randint(0, self.counts[s] - 1)
        else:
            image = idx
        return (image,) + _flat(_jitter_row(None))


class ClusterDraws:
    """The random calls of ClusterDataset.__getitem__ (cluster_dataset.py:245-275) over n images: with probs (the gating
    targets' column of cluster >= 0) the image is img_sampler.sample(), then the jitter's get_params (cluster_jitter)."""

    def __init__(self, n: int, probs=None, jitter=None):
        import torch
        _check_jitter(jitter)
        self.n, self.jitter = int(n), jitter
        self.sampler = None if probs is None else torch.distributions.categorical.Categorical(probs=torch.as_tensor(probs))

    def __len__(self):
        return self.n

    def __getitem__(self, idx):
        if self.sampler is not None:
            idx = int(self.sampler.sample())
        return (idx,) + _flat(_jitter_row(self.jitter))


def _flat(j):
    n, ops, factors = j
    return (n, *ops, *factors)


def cluster_jitter(training: bool = True):
    """ClusterDataset's ColorJitter (cluster_dataset.py:186-189)."""
    from torchvision import transforms
    if training:
        return transforms.ColorJitter(brightness=0.2, contrast=0.2, saturation=[0, 0])
    return transforms.ColorJitter(saturation=[0, 0])


def make_plan(draws, group_of, batch: int = 1, shuffle: bool = True, shift: bool = True, max_shift: int = MAX_SHIFT) -> Plan:
    """One epoch of the reference loop's draws: a DataLoader(draws, batch_size=batch, shuffle=shuffle, num_workers=0) is
    iterated (its sampler's permutation and the dataset's calls), and after each batch util.random_shift's two
    random.randint(-max_shift, max_shift) are drawn (shift=False: the test loops, which do not shift).  group_of: the shape
    group of each image; every step's images must share one (as a DataLoader batch must share a shape)."""
    import torch
    _check_jitter(getattr(draws, "jitter", None))
    loader = torch.utils.data.DataLoader(draws, batch_size=int(batch), shuffle=shuffle, num_workers=0)
    group_of = np.asarray(group_of)
    rows, groups = [], []
    for items in loader:
        image = items[0].numpy().astype(np.int64)
        n = len(image)
        padX, padY = (random.randint(-max_shift, max_shift), random.randint(-max_shift, max_shift)) if shift else (0, 0)
        g = set(int(v) for v in group_of[image])
        if len(g) != 1:
            raise ValueError(f"a step of images {image.tolist()} mixes shape groups {sorted(g)}: use batch=1")
        r = np.zeros(n, api.DATA_ROW)
        r["image"], r["padX"], r["padY"] = image, padX, padY
        r["n_ops"] = items[1].numpy()
        r["ops"] = torch.stack(list(items[2:5]), 1).numpy()
        r["factors"] = torch.stack(list(items[5:8]), 1).numpy().astype(np.float32)
        rows.append(r)
        groups.append(g.pop())
    return Plan(np.concatenate(rows) if rows else np.zeros(0, api.DATA_ROW), groups, int(batch))


# ------------------------------------------------------------------------------------------------
# readers of the reference's folder layout (decode and resize on the host, once)
# ------------------------------------------------------------------------------------------------
def _listed(d: str) -> list:
    return sorted(d + f for f in os.listdir(d))


def load_image(path: str, imsize: int):
    """Decodes with Pillow, copies a gray image into three channels and resizes with transforms.Resize(imsize), as the
    datasets' image_transform does before its colour steps; returns (uint8 [H,W,3], imsize / min(h, w))."""
    from PIL import Image
    from torchvision import transforms
    with Image.open(path) as im:
        a = rgb_image(np.asarray(im))
    scale = imsize / min(a.shape[0:2])
    resized = transforms.Resize(imsize)(transforms.ToPILImage()(a))
    return np.ascontiguousarray(np.asarray(resized, np.uint8)), scale


def from_room_folders(root_dir: str, training: bool = True, imsize: int = 480, normalize_mean: bool = True,
                      grid_cell_size: int = 5, env_list: str = "env_list.txt", storage: str = "device", **kw):
    """A RoomDataset (room_dataset.py:24-103) as a DeviceImageSet: every scene of env_list (with its optional centre), its
    rgb/, poses/, calibration/ and (training) init/ files sorted; poses and valid ground-truth cells moved by the scene's
    mean-and-grid offset with the reference's float32 torch ops (:164-207).  set.scene_counts feeds RoomDraws."""
    import torch
    with open(env_list, "r") as f:
        environment = f.readlines()
    scenes = []
    means = torch.zeros((len(environment), 3))
    for i, line in enumerate(environment):
        line = line.split()
        scenes.append(line[0])
        if len(line) > 1:
            means[i, 0], means[i, 1], means[i, 2] = float(line[1]), float(line[2]), float(line[3])
    images, poses, focal, scene_ids, gts, counts = [], [], [], [], [], []
    grid_size = math.ceil(math.sqrt(len(scenes)))
    for s, scene in enumerate(scenes):
        base = scene + "/" + root_dir
        rgb, pose_f, calib = _listed(base + "/rgb/"), _listed(base + "/poses/"), _listed(base + "/calibration/")
        init = _listed(base + "/init/") if training else None
        counts.append(len(rgb))
        offset = means[s].clone()
        if not normalize_mean:
            offset.fill_(0)
        row, col = math.ceil((s + 1) / grid_size) - 1, s % grid_size
        offset[0] += row * grid_cell_size
        offset[1] += col * grid_cell_size
        for j in range(len(rgb)):
            image, scale = load_image(rgb[j], imsize)
            images.append(image)
            focal.append(float(np.loadtxt(calib[j])) * scale)
            gt_pose = torch.from_numpy(np.loadtxt(pose_f[j])).float()
            gt_pose[0:3, 3] -= offset.float()
            poses.append(gt_pose)
            scene_ids.append(s)
            if training:
                gt_coords = torch.load(init[j])
                size = gt_coords.size()
                gt_coords = gt_coords.view(3, -1)
                mask = gt_coords.abs().sum(0) == 0
                gt_coords = gt_coords - offset.unsqueeze(1).expand(gt_coords.size()).float()
                if mask.sum() > 0:
                    gt_coords[:, mask] = 0
                gts.append(gt_coords.view(size))
    ds = DeviceImageSet(images, torch.stack(poses), focal, scene_ids, gt=gts if training else None, mean=ROOM_MEAN,
                        std=ROOM_STD, storage=storage, **kw)
    ds.scene_counts = counts
    return ds


def from_cluster_folder(root_dir: str, training: bool = True, imsize: int = 480, env_list: str = "env_list.txt",
                        storage: str = "device", attachments=None, **kw):
    """A ClusterDataset's images (cluster_dataset.py:170-214) as a DeviceImageSet: the one environment of env_list, its
    rgb/, poses/, calibration/ and (training) init/ files sorted, no offset, scene -1.  Its jitter is cluster_jitter's,
    drawn by ClusterDraws; attachments (a gating-target row per image, for init_gating.py -c) as DeviceImageSet takes them."""
    import torch
    with open(env_list, "r") as f:
        environment = f.readlines()
    if len(environment) > 1:
        raise ValueError("env_list holds more than one environment; clustering supports one")
    base = environment[0].strip() + "/" + root_dir
    rgb, pose_f, calib = _listed(base + "/rgb/"), _listed(base + "/poses/"), _listed(base + "/calibration/")
    images, focal = [], []
    for j in range(len(rgb)):
        image, scale = load_image(rgb[j], imsize)
        images.append(image)
        focal.append(float(np.loadtxt(calib[j])) * scale)
    poses = torch.stack([torch.from_numpy(np.loadtxt(p)).float() for p in pose_f])
    gts = [torch.load(f) for f in _listed(base + "/init/")] if training else None
    return DeviceImageSet(images, poses, focal, [-1] * len(images), gt=gts, attachments=attachments, mean=CLUSTER_MEAN,
                          std=CLUSTER_STD, storage=storage, **kw)
