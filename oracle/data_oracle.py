"""The reference's item path on the host, for the tests of esac_b200.data (not a product path).

pil_item: one plan row's image through PIL / torchvision as the datasets' image_transform and util.random_shift run it
(ColorJitter's ops in the row's order, ToTensor, Normalize, nn.ZeroPad2d).  restate_item: the same in numpy float32, the
arithmetic the kernels state (blend a + f (b - a) with no contraction, PIL's fixed-point luma, the contrast grey
int(sum / N + 0.5)).  room_offset: room_dataset.py:164-207.  reference_loop: the reference training / test loop's random
calls, made by the datasets' own code shapes (a real ColorJitter transform on a small image, random.choice / randint,
Categorical.sample, a shuffling DataLoader and util.random_shift), recording what each step drew.
"""
from __future__ import annotations

import math
import random

import numpy as np
import torch
import torch.nn as nn
from PIL import Image
from torchvision import transforms
from torchvision.transforms import functional as F

BRIGHTNESS, CONTRAST, SATURATION = 0, 1, 2


def _row_ops(row):
    n = int(row["n_ops"])
    return [(int(row["ops"][k]), float(row["factors"][k])) for k in range(n)]


def pil_item(image: np.ndarray, row, mean, std) -> torch.Tensor:
    """uint8 [H,W,3] -> float32 [3,H,W]: jitter (PIL), ToTensor, Normalize, ZeroPad2d((padX, -padX, padY, -padY))."""
    img = transforms.ToPILImage()(image)
    for op, f in _row_ops(row):
        img = (F.adjust_brightness, F.adjust_contrast, F.adjust_saturation)[op](img, f)
    t = transforms.Normalize(mean=[mean] * 3 if np.ndim(mean) == 0 else list(mean),
                             std=[std] * 3 if np.ndim(std) == 0 else list(std))(transforms.ToTensor()(img))
    padX, padY = int(row["padX"]), int(row["padY"])
    return nn.ZeroPad2d((padX, -padX, padY, -padY))(t.unsqueeze(0))[0]


def luma(a: np.ndarray) -> np.ndarray:
    a = a.astype(np.int64)
    return ((a[..., 0] * 19595 + a[..., 1] * 38470 + a[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def blend(a, b, f) -> np.ndarray:
    """Image.blend(a, b, f) per channel: float32 a + f (b - a), truncated for 0 <= f <= 1, else clipped then truncated."""
    al = np.float32(f)
    with np.errstate(over="ignore"):
        t = np.asarray(a, np.float32) + al * (np.asarray(b, np.float32) - np.asarray(a, np.float32))
    if 0.0 <= al <= 1.0:
        return t.astype(np.uint8)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, t)).astype(np.uint8)


def jitter(image: np.ndarray, ops) -> np.ndarray:
    img = image
    for op, f in ops:
        if op == BRIGHTNESS:
            img = blend(np.zeros_like(img), img, f)
        elif op == CONTRAST:
            L = luma(img)
            m = int(float(L.astype(np.int64).sum()) / L.size + 0.5)
            img = blend(np.full_like(img, m), img, f)
        else:
            img = blend(np.repeat(luma(img)[..., None], 3, -1), img, f)
    return img


def normalize(u: np.ndarray, mean, std) -> np.ndarray:
    """ToTensor + Normalize: (u / 255 - m) / s in float32, u uint8 [..., 3] -> float32 [3, ...]."""
    m = np.asarray(np.broadcast_to(np.float32(mean), (3,)), np.float32)
    s = np.asarray(np.broadcast_to(np.float32(std), (3,)), np.float32)
    x = np.moveaxis(u.astype(np.float32), -1, 0) / np.float32(255)
    return (x - m.reshape((3,) + (1,) * (x.ndim - 1))) / s.reshape((3,) + (1,) * (x.ndim - 1))


def restate_item(image: np.ndarray, row, mean, std) -> np.ndarray:
    v = normalize(jitter(image, _row_ops(row)), mean, std)
    H, W = image.shape[:2]
    padX, padY = int(row["padX"]), int(row["padY"])
    out = np.zeros_like(v)   # out[y][x] = v[y - padY][x - padX], zero outside
    y0, y1, x0, x1 = max(0, padY), min(H, H + padY), max(0, padX), min(W, W + padX)
    if y0 < y1 and x0 < x1:
        out[:, y0:y1, x0:x1] = v[:, y0 - padY:y1 - padY, x0 - padX:x1 - padX]
    return out


def room_offset(gt_pose: torch.Tensor, gt_coords, means_row: torch.Tensor, scene_idx: int, n_scenes: int,
                grid_cell_size: int = 5, normalize_mean: bool = True):
    """room_dataset.py:164-207 on a float32 [4,4] pose and a float32 [3,h,w] map (or None)."""
    gt_pose = gt_pose.clone()
    offset = means_row.clone()
    if not normalize_mean:
        offset.fill_(0)
    grid_size = math.ceil(math.sqrt(n_scenes))
    row = math.ceil((scene_idx + 1) / grid_size) - 1
    col = scene_idx % grid_size
    offset[0] += row * grid_cell_size
    offset[1] += col * grid_cell_size
    gt_pose[0:3, 3] -= offset.float()
    if gt_coords is None:
        return gt_pose, None
    gt_coords_size = gt_coords.size()
    gt_coords = gt_coords.reshape(3, -1)
    coords_mask = gt_coords.abs().sum(0) == 0
    offset = offset.unsqueeze(1).expand(gt_coords.size())
    gt_coords = gt_coords - offset.float()
    if coords_mask.sum() > 0:
        gt_coords[:, coords_mask] = 0
    return gt_pose, gt_coords.view(gt_coords_size)


class _Recorder(transforms.ColorJitter):
    """ColorJitter that records what its forward drew."""

    def forward(self, img):
        params = self.get_params(self.brightness, self.contrast, self.saturation, self.hue)
        self.drawn.append(params)
        fn_idx, b, c, s, h = params
        for fn_id in fn_idx:
            if fn_id == 0 and b is not None:
                img = F.adjust_brightness(img, b)
            elif fn_id == 1 and c is not None:
                img = F.adjust_contrast(img, c)
            elif fn_id == 2 and s is not None:
                img = F.adjust_saturation(img, s)
        return img


class _RoomItems(torch.utils.data.Dataset):
    """RoomDataset.__getitem__'s index mapping (room_dataset.py:134-149) over scenes of the given image counts."""

    def __init__(self, counts, scene, training):
        self.scenes = [f"scene{i}" for i in range(len(counts))]
        self.files = {s: list(range(c)) for s, c in zip(self.scenes, counts)}
        self.starts = dict(zip(self.scenes, np.concatenate([[0], np.cumsum(counts)[:-1]]).tolist()))
        self.scene, self.training, self.cnt = scene, training, int(sum(counts))

    def __len__(self):
        if self.scene >= 0:
            return len(self.files[self.scenes[self.scene]])
        return 1000 if self.training else self.cnt

    def __getitem__(self, global_idx):
        if self.scene >= 0:
            local_idx, scene = global_idx, self.scenes[self.scene]
        elif self.training:
            scene = random.choice(self.scenes)
            local_idx = random.randint(0, len(self.files[scene]) - 1)
        else:
            return global_idx, torch.zeros(3, 4, 4)
        return self.starts[scene] + local_idx, torch.zeros(3, 4, 4)


class _ClusterItems(torch.utils.data.Dataset):
    """ClusterDataset.__getitem__'s draws (cluster_dataset.py:262-270) with its image_transform on a small image."""

    def __init__(self, n, probs, jitter):
        self.n = n
        self.img_sampler = None if probs is None else torch.distributions.categorical.Categorical(probs=probs)
        self.jitter = _Recorder()
        # the ranges the given transform's constructor checked, as get_params takes them
        self.jitter.brightness, self.jitter.contrast, self.jitter.saturation = jitter.brightness, jitter.contrast, jitter.saturation
        self.jitter.hue = jitter.hue
        self.jitter.drawn = []
        self.image = Image.fromarray(np.arange(4 * 6 * 3, dtype=np.uint8).reshape(4, 6, 3))

    def __len__(self):
        return self.n

    def __getitem__(self, idx):
        if self.img_sampler is not None:
            idx = int(self.img_sampler.sample())
        image = transforms.ToTensor()(self.jitter(self.image))
        return idx, image


def reference_loop(kind: str, steps: int, counts=None, scene=-1, training=True, n=None, probs=None, jitter=None,
                   shuffle=True, shift=True):
    """The first `steps` steps of the reference loop (batch 1) over a room set (kind "room": counts per scene, scene,
    training) or a clustered set (kind "cluster": n images, probs, jitter): per step (image, padX, padY, jitter draw or
    None).  The loop pads the item's image with util.random_shift's draws, as the training scripts do."""
    from esac_b200.compat import OUTPUT_SUBSAMPLE, random_shift
    ds = _RoomItems(counts, scene, training) if kind == "room" else _ClusterItems(n, probs, jitter)
    loader = torch.utils.data.DataLoader(ds, shuffle=shuffle, num_workers=0)
    out = []
    for i, (idx, image) in enumerate(loader):
        if i == steps:
            break
        padX = padY = 0
        if shift:
            padX, padY, _ = random_shift(image, int(OUTPUT_SUBSAMPLE / 2))
        drawn = ds.jitter.drawn[-1] if kind == "cluster" else None
        out.append((int(idx), padX, padY, drawn))
    return out
