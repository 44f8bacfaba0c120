"""Clustering a large environment into experts on the device: the replacement of ClusterDataset.__cluster__ and its soft
gating targets (code/cluster_dataset.py:37-140, 219-240).

    c = cluster_environment(init_maps, num_clusters=20)
    c.gating_probs        # [N, K] float32: init_gating.py -c's KLDivLoss target, the draw weights of one cluster's images

The per-image statistics (api.cluster_statistics), each 2-means split (api.kmeans2) and the centres, sizes and targets
(api.cluster_targets) run on the GPU; this host driver keeps the hierarchy: a list of clusters, the largest popped and
split in two until there are num_clusters.  The numbering of the clusters is this implementation's: the 2-means has its
own random stream, not cv::RNG's, so a split may come out with its halves the other way round from cv2.kmeans.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import api


@dataclass
class Clustering:
    cam_centers: torch.Tensor   # float32 [K,3]: mean of each cluster's image means
    cam_sizes: torch.Tensor     # float32 [K,1]: mean squared distance of those means to the centre
    labels: torch.Tensor        # int64 [N]: each image's cluster
    gating_probs: torch.Tensor  # float32 [N,K]: soft gating targets
    medians: torch.Tensor       # float32 [N,3]: each image's median scene coordinate (what the 2-means splits)
    means: torch.Tensor         # float32 [N,3]: each image's mean scene coordinate
    counts: torch.Tensor        # int32 [N]: each image's valid cells


def hierarchy(n: int, num_clusters: int, split_fn) -> np.ndarray:
    """The hierarchy of cluster_dataset.py:64-102 over n images: clusters (indices, label) in a list; the first (largest)
    is popped and split_fn(indices, split) gives its 0 / 1 labels; label 0 keeps the parent's label, label 1 takes the
    next counter value; the list is then stable-sorted by size, descending.  Returns the n labels (int64)."""
    labels = np.zeros(n, np.int64)
    clusters = [(np.arange(n), 0)]
    counter = 0
    while len(clusters) < num_clusters:
        idx, label = clusters.pop(0)
        if len(idx) < 2:
            raise RuntimeError(f"cluster_environment: the largest cluster ({label}) holds only image {int(idx[0])}, "
                               f"and {num_clusters} clusters need it split; use fewer clusters")
        counter += 1
        half = np.asarray(split_fn(idx, counter - 1))
        clusters.append((idx[half == 0], label))
        clusters.append((idx[half == 1], counter))
        labels[idx[half == 1]] = counter
        clusters.sort(key=lambda c: len(c[0]), reverse=True)
    return labels


def cluster_environment(init_maps, num_clusters: int, softness: float = 5.0, seed: int = 0,
                        device: torch.device | None = None) -> Clustering:
    """Clusters N training images by their ground-truth maps (init_maps: a stacked float32 [N,3,H,W] or a list of N
    [3,H_b,W_b], host or CUDA) into num_clusters experts.  Each split is a 2-means of the images' median scene coordinates
    (10 attempts, 100 iterations, eps 0.1 m, as cluster_dataset.py:65); split s draws from (seed, s).  Raises, naming the
    images, when a map has no valid cell or a non-finite median or mean, or when a cluster to split holds one image.
    `device`: where the clustering runs when the maps are on the host (default: the current CUDA device)."""
    medians, means, counts, status = api.cluster_statistics(init_maps)
    st = status.cpu().numpy()
    if st.any():
        bad = np.flatnonzero(st)
        kinds = {1: "no valid cell", 2: "a non-finite median or mean"}
        listed = ", ".join(f"{int(i)} ({kinds[int(st[i])]})" for i in bad[:10])
        raise RuntimeError(f"cluster_environment: {len(bad)} image(s) cannot be clustered: {listed}"
                           + (", ..." if len(bad) > 10 else ""))
    N = int(medians.shape[0])
    K = int(num_clusters)
    if not 1 <= K <= min(N, api.MAX_CLUSTERS):
        raise RuntimeError(f"cluster_environment: num_clusters={num_clusters} outside [1, {min(N, api.MAX_CLUSTERS)}] "
                           f"for {N} images")
    if not medians.is_cuda:
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        medians, means, counts = medians.to(dev), means.to(dev), counts.to(dev)

    def split(idx, s):
        pts = medians[torch.from_numpy(idx).to(medians.device)].contiguous()
        half, _, _ = api.kmeans2(pts, seed, split=s)
        return half.cpu().numpy()

    labels = torch.from_numpy(hierarchy(N, K, split)).to(medians.device)
    centres, sizes, probs = api.cluster_targets(means, labels, K, softness)
    return Clustering(centres, sizes, labels, probs, medians, means, counts)
