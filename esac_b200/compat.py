"""Caller-side shims (SURVEY.md 8f rank 3) that let the reference's training / test loop logic run in this image.

Nothing here is on the hot path.  Two things the unchanged callers need and this image cannot give them:

* `util.random_shift` (code/util.py:4-11) passes `Expert.OUTPUT_SUBSAMPLE / 2` (a float) to `random.randint`, which is a
  TypeError from Python 3.12 on; `random_shift` below is the same augmentation with the bound converted to int.
* `RoomDataset` / `ClusterDataset` (code/room_dataset.py, code/cluster_dataset.py) need scikit-image and dataset files on
  disk; `SyntheticRoomDataset` yields the same 6-tuple `(index, image, focallength, gt_pose, gt_coords, expert)`
  (room_dataset.py:214) from `esac_b200.synth.make_scene`, so `DataLoader(dataset, shuffle=True)` and the loops of
  train_esac.py:96-185 / test_esac.py:137-230 / ref_expert.py:95-160 run as written.  `SyntheticClusterDataset` stands in
  for `ClusterDataset`: one large environment, clustered on the device by `esac_b200.cluster.cluster_environment`.

The synthetic "experts" that stand in for the CNNs read the scene coordinates the dataset attaches to every sample
(`dataset.prediction_for(index)`): the networks themselves are out of scope (SURVEY.md section 2, rows 9-17).
"""
from __future__ import annotations

import random

import numpy as np
import torch
import torch.nn as nn
from torch.utils.data import Dataset

from .synth import make_scene, rodrigues

OUTPUT_SUBSAMPLE = 8  # code/expert.py:13


def random_shift(image: torch.Tensor, max_shift):
    """util.random_shift (code/util.py:4-11): zero-pad shift by (padX, padY) in [-max_shift, max_shift]."""
    max_shift = int(max_shift)
    padX = random.randint(-max_shift, max_shift)
    padY = random.randint(-max_shift, max_shift)
    pad = nn.ZeroPad2d((padX, -padX, padY, -padY))
    return padX, padY, pad(image)


class SyntheticRoomDataset(Dataset):
    """Stand-in for RoomDataset: `num_experts` rooms on the reference's 5 m grid (room_dataset.py:177-184), `length`
    images of 640x480 px, each with a ground-truth pose, ground-truth scene coordinates [3,60,80] and the id of the room it
    was taken in.  Deterministic in (seed, index).  gt_valid_frac < 1 zeroes a deterministic share of 1 - gt_valid_frac
    of the ground-truth cells (cells without ground truth, as in the sparse SfM datasets)."""

    def __init__(self, num_experts: int = 4, length: int = 16, hypotheses: int = 256, seed: int = 0, training: bool = True,
                 image_hw=(480, 640), outlier_frac: float = 0.4, noise: float = 0.02, gt_valid_frac: float = 1.0):
        self.num_experts = num_experts
        self.gt_valid_frac = gt_valid_frac
        self.length = length
        self.hypotheses = hypotheses
        self.seed = seed
        self.training = training
        self.image_hw = image_hw
        self.outlier_frac = outlier_frac
        self.noise = noise
        self._cache = {}

    def __len__(self):
        return self.length

    def scene(self, index: int):
        if index not in self._cache:
            H, W = self.image_hw[0] // OUTPUT_SUBSAMPLE, self.image_hw[1] // OUTPUT_SUBSAMPLE
            self._cache[index] = make_scene(E=self.num_experts, H=H, W=W, M=self.hypotheses, sub=OUTPUT_SUBSAMPLE,
                                            seed=self.seed * 100003 + index, outlier_frac=self.outlier_frac, noise=self.noise,
                                            active_only=False)
        return self._cache[index]

    def prediction_for(self, index: int) -> torch.Tensor:
        """What a trained ensemble would predict for image `index`: [E,3,60,80] float32 (GT expert: noisy truth with
        outliers; the others: points around their own room)."""
        return torch.from_numpy(self.scene(index).coords)

    def __getitem__(self, index: int):
        sc = self.scene(index)
        rng = np.random.default_rng(self.seed * 7919 + index)
        image = torch.from_numpy(rng.random((1, *self.image_hw), dtype=np.float32))   # grayscale, room_dataset.py:60-66
        gt_pose = torch.from_numpy(sc.gt_pose.copy())
        if self.training:
            gt_coords = torch.from_numpy(sc.coords[sc.gt_expert].copy())
            if self.gt_valid_frac < 1.0:
                # cells without ground truth are all zero (sparse SfM depth, Aachen / Dubrovnik); own stream, so the image
                # and the kept cells do not change
                drop = np.random.default_rng(self.seed * 6151 + index).random(gt_coords.shape[1:]) >= self.gt_valid_frac
                gt_coords[:, torch.from_numpy(drop)] = 0.0
        else:
            gt_coords = 0                                                              # room_dataset.py:209-212
        return index, image, float(sc.f), gt_pose, gt_coords, int(sc.gt_expert)


class SyntheticClusterDataset(Dataset):
    """Stand-in for ClusterDataset (cluster_dataset.py:145-289): one connected outdoor environment `extent` metres across,
    `length` images taken from cameras at 1.6 m height anywhere in it, looking horizontally in any direction, each with a
    ground-truth pose and sparse ground-truth scene coordinates (a share gt_valid_frac of the cells; the rest all zero, as
    in the SfM-based Aachen / Dubrovnik maps) of [3,60,80] for a landscape image and [3,80,60] for a portrait one (a share
    portrait_frac).  Yields the reference's 6-tuple with expert -1.  Deterministic in (seed, index).

    With training=True the environment is clustered into num_clusters experts at construction, on the device
    (esac_b200.cluster.cluster_environment), and cam_centers, cam_sizes, labels and gating_probs are exposed as the
    reference's are; with cluster >= 0, every item is an image drawn with probability gating_probs[:, cluster]
    (cluster_dataset.py:242-243, 266-267), whatever index is asked for."""

    def __init__(self, num_clusters: int = 10, length: int = 200, cluster: int = -1, training: bool = True,
                 softness: float = 5.0, seed: int = 0, extent: float = 300.0, gt_valid_frac: float = 0.5,
                 portrait_frac: float = 0.3, focal_length: float = 525.0):
        self.num_experts = num_clusters
        self.length = length
        self.cluster = cluster
        self.training = training
        self.softness = softness
        self.seed = seed
        self.extent = extent
        self.gt_valid_frac = gt_valid_frac
        self.portrait_frac = portrait_frac
        self.focal_length = focal_length
        if training:
            from .cluster import cluster_environment
            c = cluster_environment([self.init_map(i) for i in range(length)], num_clusters, softness=softness, seed=seed)
            self.clustering = c
            self.cam_centers, self.cam_sizes, self.labels, self.gating_probs = c.cam_centers, c.cam_sizes, c.labels, c.gating_probs
            if cluster >= 0:
                self.img_sampler = torch.distributions.categorical.Categorical(probs=self.gating_probs[:, cluster].cpu())

    def __len__(self):
        return self.length

    def portrait(self, index: int) -> bool:
        return bool(np.random.default_rng([self.seed, index, 1]).random() < self.portrait_frac)

    def pose(self, index: int) -> np.ndarray:
        """Camera -> world, float32 [4,4]: a camera at 1.6 m height, yaw uniform, pitch within +-5 degrees."""
        rng = np.random.default_rng([self.seed, index, 2])
        centre = np.array([rng.uniform(0, self.extent), rng.uniform(0, self.extent), 1.6])
        yaw, pitch = rng.uniform(0, 2 * np.pi), rng.uniform(-np.pi / 36, np.pi / 36)
        look = rodrigues([0.0, 0.0, yaw]) @ rodrigues([pitch, 0.0, 0.0])
        # camera axes: x right, y down, z forward; forward along the world's +y before the yaw, up the world's +z
        base = np.array([[1.0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]]).T
        T = np.eye(4)
        T[:3, :3] = look @ base
        T[:3, 3] = centre
        return T.astype(np.float32)

    def init_map(self, index: int) -> torch.Tensor:
        """Ground-truth scene coordinates [3,H,W] (H, W = 60, 80 or 80, 60): depths 3-40 m through the pose, cells without
        ground truth all zero."""
        H, W = (80, 60) if self.portrait(index) else (60, 80)
        rng = np.random.default_rng([self.seed, index, 3])
        xs = np.arange(W) * OUTPUT_SUBSAMPLE + OUTPUT_SUBSAMPLE // 2 - W * OUTPUT_SUBSAMPLE / 2
        ys = np.arange(H) * OUTPUT_SUBSAMPLE + OUTPUT_SUBSAMPLE // 2 - H * OUTPUT_SUBSAMPLE / 2
        px, py = np.meshgrid(xs, ys)
        depth = rng.uniform(3.0, 40.0, (H, W))
        cam = np.stack([px / self.focal_length * depth, py / self.focal_length * depth, depth]).reshape(3, -1)
        T = self.pose(index).astype(np.float64)
        world = (T[:3, :3] @ cam + T[:3, 3:]).reshape(3, H, W).astype(np.float32)
        world[:, rng.random((H, W)) >= self.gt_valid_frac] = 0.0
        return torch.from_numpy(world)

    def __getitem__(self, index: int):
        if self.cluster >= 0 and self.training:
            index = int(self.img_sampler.sample())
        H, W = (80, 60) if self.portrait(index) else (60, 80)
        rng = np.random.default_rng([self.seed, index, 4])
        image = torch.from_numpy(rng.random((1, H * OUTPUT_SUBSAMPLE, W * OUTPUT_SUBSAMPLE), dtype=np.float32))
        gt_coords = self.init_map(index) if self.training else 0
        return index, image, float(self.focal_length), torch.from_numpy(self.pose(index)), gt_coords, -1
