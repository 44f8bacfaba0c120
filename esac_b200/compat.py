"""Caller-side shims (SURVEY.md 8f rank 3) that let the reference's training / test loop logic run in this image.

Nothing here is on the hot path.  Two things the unchanged callers need and this image cannot give them:

* `util.random_shift` (code/util.py:4-11) passes `Expert.OUTPUT_SUBSAMPLE / 2` (a float) to `random.randint`, which is a
  TypeError from Python 3.12 on; `random_shift` below is the same augmentation with the bound converted to int.
* `RoomDataset` / `ClusterDataset` (code/room_dataset.py, code/cluster_dataset.py) need scikit-image and dataset files on
  disk; `SyntheticRoomDataset` yields the same 6-tuple `(index, image, focallength, gt_pose, gt_coords, expert)`
  (room_dataset.py:214) from `esac_b200.synth.make_scene`, so `DataLoader(dataset, shuffle=True)` and the loops of
  train_esac.py:96-185 / test_esac.py:137-230 / ref_expert.py:95-160 run as written.

The synthetic "experts" that stand in for the CNNs read the scene coordinates the dataset attaches to every sample
(`dataset.prediction_for(index)`): the networks themselves are out of scope (SURVEY.md section 2, rows 9-17).
"""
from __future__ import annotations

import random

import numpy as np
import torch
import torch.nn as nn
from torch.utils.data import Dataset

from .synth import make_scene

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
