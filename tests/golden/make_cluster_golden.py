"""Writes tests/golden/cluster/cluster_*.npz: small clustered environments and what the reference route makes of them.

The reference route is ClusterDataset.__cluster__ and its gating targets (cluster_dataset.py:37-140, 219-240), restated
here because that module cannot be imported without scikit-image: per image, torch's valid-cell mask, torch.median and
sum / count; the hierarchy (pop the largest cluster, split it with cv2.kmeans(points, 2, None, (EPS + MAX_ITER, 100, 0.1),
10, KMEANS_PP_CENTERS), label 0 keeps the parent's label, label 1 takes the next one, stable sort by size, descending);
then the centres, sizes and targets in torch float32.

Each environment is a hierarchy of well separated blobs of image medians, with distinct cluster sizes at every split, so
any sound 2-means finds the same partitions: a test compares partitions up to renumbering.

    python tests/golden/make_cluster_golden.py      (needs cv2)
"""
from __future__ import annotations

import math
from pathlib import Path

import cv2
import numpy as np
import torch

HERE = Path(__file__).resolve().parent / "cluster"   # apart from the oracle's fixtures, which test_oracle.py globs

# (name, K, blobs: (centre, images), map shapes cycled over the images)
ENVIRONMENTS = [
    ("cluster_k4_ragged", 4, [((0, 0, 0), 9), ((40, 0, 2), 8), ((400, 30, 0), 7), ((440, 30, 1), 6)],
     [(6, 8), (8, 6), (6, 11)]),
    ("cluster_k5", 5, [((0, 0, 0), 11), ((0, 60, 0), 10), ((300, 0, 5), 9), ((300, 70, 5), 8), ((150, 600, 0), 12)],
     [(5, 7)]),
]


def make_maps(blobs, shapes, seed):
    rng = np.random.default_rng(seed)
    maps = []
    for centre, count in blobs:
        for _ in range(count):
            H, W = shapes[len(maps) % len(shapes)]
            m = (np.asarray(centre, np.float64)[:, None, None] + rng.normal(0, 1.5, (3, H, W))).astype(np.float32)
            m[:, rng.random((H, W)) < 0.3] = 0.0           # cells without ground truth
            maps.append(m)
    order = rng.permutation(len(maps))                    # blobs interleaved in file order
    return [maps[i] for i in order]


def reference_route(maps, K, softness=5.0):
    stats = []
    for m in maps:
        d = torch.from_numpy(m).view(3, -1)
        mask = d.sum(0) != 0
        d = d[:, mask]
        stats.append((d.median(1)[0], d.sum(1) / mask.sum()))
    medians = torch.stack([s[0] for s in stats]).numpy()
    means = torch.stack([s[1] for s in stats])
    criteria = (cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 100, 0.1)
    labels = np.zeros(len(maps))
    clusters = [(medians, 0)]
    counter = 0
    while len(clusters) < K:
        points, label = clusters.pop(0)
        counter += 1
        _, half, _ = cv2.kmeans(points, 2, None, criteria, 10, cv2.KMEANS_PP_CENTERS)
        half = half[:, 0]
        clusters.append((points[half == 0], label))
        clusters.append((points[half == 1], counter))
        mine = labels[labels == label]
        mine[half == 1] = counter
        labels[labels == label] = mine
        clusters = sorted(clusters, key=lambda c: c[0].shape[0], reverse=True)
    centres = torch.zeros(K, 3)
    sizes = torch.zeros(K, 1)
    for k in range(K):
        data = means[torch.from_numpy(labels == k)]
        centres[k] = data.mean(0)
        sizes[k] = ((data - centres[k].unsqueeze(0).expand(len(data), 3)).norm(dim=1) ** 2).mean()
    probs = torch.zeros(len(maps), K)
    for i in range(len(maps)):
        d = means[i].unsqueeze(0).expand(centres.size()) - centres
        d = d.norm(dim=1) ** 2
        d = d / sizes[:, 0] / 2
        d = torch.exp(-d * softness)
        d /= torch.sqrt(2 * math.pi * sizes[:, 0])
        d /= d.sum() + 0.0000001
        probs[i] = d
    return dict(labels=labels.astype(np.int64), cam_centers=centres.numpy(), cam_sizes=sizes.numpy(),
                gating_probs=probs.numpy(), medians=medians, means=means.numpy())


def main():
    cv2.setRNGSeed(1305)
    for n, (name, K, blobs, shapes) in enumerate(ENVIRONMENTS):
        maps = make_maps(blobs, shapes, 7 + n)
        ref = reference_route(maps, K)
        arrays = {f"map_{i}": m for i, m in enumerate(maps)}
        np.savez_compressed(HERE / f"{name}.npz", K=K, n_maps=len(maps), **arrays, **ref)
        print(name, len(maps), "maps, sizes", np.bincount(ref["labels"]).tolist())


if __name__ == "__main__":
    main()
