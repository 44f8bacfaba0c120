"""Oracle for clustering a large environment into experts (cluster_dataset.py:19-140, 219-240).  TEST INFRASTRUCTURE ONLY.

A float64 numpy restatement of esac_b200/csrc/cluster.cu and of the host driver esac_b200/cluster.py:

* statistics: the valid cells ((x + y) + z != 0 in float32), each coordinate's lower median sorted[(n-1)//2] in the
  order of the float's order-preserving integer key (so -0 sorts before +0), the first NaN when there is one, and the
  fp64 mean rounded to float32;
* kmeans2: k-means++ seeding with 3 trials and Lloyd iterations on the same mix64 stream, with every sum taken in the
  kernel's fixed order -- thread t of T = 256 adds its contiguous chunk of ceil(n/T) points in index order, then
  partial[t] += partial[t + s] for s = T/2 .. 1 -- so the labels agree exactly and the rest to the last bit or so;
* targets: the centres, sizes and soft gating targets in float64;
* cluster_environment: the hierarchy of cluster_dataset.py:64-102.

Only tests/ may import this module; the product path never does.
"""
from __future__ import annotations

import numpy as np

from oracle.esac_oracle import _GOLD, mix64

T = 256                 # threads of a k-means CTA: the shape of every k-means reduction (kKmeansThreads)
STATUS_OK, STATUS_EMPTY, STATUS_NONFINITE = 0, 1, 2


# ---- per-image statistics ----------------------------------------------------------------------------------------------
def _key(v: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(v, np.float32).view(np.uint32)
    return u ^ np.where(u >> 31 == 1, np.uint32(0xFFFFFFFF), np.uint32(0x80000000))


def statistics(m) -> tuple:
    """One map [3,H,W] float32: (median float32 [3], mean float32 [3], count, status)."""
    v = np.asarray(m, np.float32).reshape(3, -1)
    valid = ((v[0] + v[1]) + v[2]) != np.float32(0)
    cells = v[:, valid]
    n = cells.shape[1]
    if n == 0:
        return np.full(3, np.nan, np.float32), np.full(3, np.nan, np.float32), 0, STATUS_EMPTY
    med = np.empty(3, np.float32)
    for c in range(3):
        row = cells[c]
        nan = np.isnan(row)
        if nan.any():
            med[c] = row[int(np.argmax(nan))]        # the first NaN, its own bits
        else:
            med[c] = row[np.argsort(_key(row), kind="stable")[(n - 1) // 2]]
    mean = (cells.astype(np.float64).sum(1) / n).astype(np.float32)
    finite = np.isfinite(med).all() and np.isfinite(mean).all()
    return med, mean, n, STATUS_OK if finite else STATUS_NONFINITE


def statistics_batch(maps) -> tuple:
    """A list of maps: (median [B,3], mean [B,3], count [B], status [B])."""
    out = [statistics(m) for m in maps]
    return (np.stack([o[0] for o in out]), np.stack([o[1] for o in out]), np.array([o[2] for o in out], np.int64),
            np.array([o[3] for o in out], np.int64))


# ---- 2-means -----------------------------------------------------------------------------------------------------------
def draw(seed: int, split: int, attempt: int, d: int) -> int:
    s = mix64(seed + _GOLD * (split + 1))
    s = mix64(s + _GOLD * (attempt + 1))
    return mix64(s + _GOLD * (d + 1))


def _chunked(vals: np.ndarray) -> np.ndarray:
    """[..., n] -> [..., T, C]: thread t's chunk, zero-padded."""
    n = vals.shape[-1]
    C = -(-n // T)
    pad = np.zeros(vals.shape[:-1] + (T * C - n,))
    return np.concatenate([vals, pad], axis=-1).reshape(vals.shape[:-1] + (T, C))


def tree_sum(vals: np.ndarray) -> tuple:
    """The kernel's sum of [..., n]: (total [...], partials [..., T])."""
    part = np.cumsum(_chunked(vals), axis=-1)[..., -1]
    r = part.copy()
    s = T // 2
    while s:
        r[..., :s] = r[..., :s] + r[..., s:2 * s]
        s //= 2
    return r[..., 0], part


def _d2(P: np.ndarray, c) -> np.ndarray:
    dx, dy, dz = P[..., 0] - c[0], P[..., 1] - c[1], P[..., 2] - c[2]
    return (dx * dx + dy * dy) + dz * dz


def _assign(P: np.ndarray, c: np.ndarray):
    """Nearer centre (0 on a tie); an empty cluster takes the point farthest from the other centre (first on a tie)."""
    n = len(P)
    d0, d1 = _d2(P, c[0]), _d2(P, c[1])
    lab = (d1 < d0).astype(np.int64)
    n1 = int(lab.sum())
    if n1 == 0 or n1 == n:
        k = 1 if n1 == 0 else 0
        lab[int(np.argmax(_d2(P, c[1 - k])))] = k
    d = np.where(lab == 1, d1, d0)
    vals = np.stack([np.where(lab == 0, P[:, 0], 0.), np.where(lab == 0, P[:, 1], 0.), np.where(lab == 0, P[:, 2], 0.),
                     np.where(lab == 1, P[:, 0], 0.), np.where(lab == 1, P[:, 1], 0.), np.where(lab == 1, P[:, 2], 0.), d])
    tot, _ = tree_sum(vals)
    n1 = int(lab.sum())
    return lab, tot[:6].reshape(2, 3), np.array([n - n1, n1], np.float64), tot[6]


def kmeans_attempt(P: np.ndarray, seed: int, split: int, attempt: int, max_iter: int, eps: float):
    """One attempt: (labels, centres fp64 [2,3], compactness)."""
    n = len(P)
    i0 = ((draw(seed, split, attempt, 0) >> 32) * n) >> 32
    dist = _d2(P, P[i0])
    sum0, part = tree_sum(dist)
    pre = np.concatenate([[0.], np.cumsum(part)])
    cum = (pre[:T, None] + np.cumsum(_chunked(dist), axis=-1)).reshape(-1)[:n]
    best, best_i = np.inf, 0
    for trial in range(3):
        p = ((draw(seed, split, attempt, 1 + trial) >> 11) * 2.0 ** -53) * sum0
        hits = np.flatnonzero(cum >= p)
        ci = min(int(hits[0]), n - 1) if len(hits) else n - 1
        pot, _ = tree_sum(np.minimum(dist, _d2(P, P[ci])))
        if pot < best:
            best, best_i = pot, ci
    c = np.stack([P[i0], P[best_i]])
    for _ in range(max_iter):
        _, sums, counts, _ = _assign(P, c)
        nc = sums / counts[:, None]
        shift = max(float(_d2(nc[k], c[k])) for k in range(2))
        c = nc
        if shift <= eps * eps:
            break
    lab, _, _, comp = _assign(P, c)
    return lab, c, float(comp)


def kmeans2(points, seed: int, attempts: int = 10, max_iter: int = 100, eps: float = 0.1, split: int = 0):
    """(labels int64 [n], centres float32 [2,3], compactness) of the attempt with the lowest compactness (first on a tie)."""
    P = np.asarray(points, np.float32).astype(np.float64)
    runs = [kmeans_attempt(P, seed, split, a, max_iter, eps) for a in range(attempts)]
    b = int(np.argmin([r[2] for r in runs]))
    return runs[b][0], runs[b][1].astype(np.float32), runs[b][2]


# ---- centres, sizes and targets ----------------------------------------------------------------------------------------
def targets(means, labels, K: int, softness: float = 5.0):
    """(cam_centers [K,3], cam_sizes [K,1], gating_probs [N,K]) in float64."""
    m = np.asarray(means, np.float32).astype(np.float64)
    labels = np.asarray(labels)
    centres = np.stack([m[labels == k].mean(0) for k in range(K)])
    sizes = np.array([(_d2(m[labels == k], centres[k])).mean() for k in range(K)])
    d2 = np.stack([_d2(m, centres[k]) for k in range(K)], 1)
    e = np.exp(-d2 / sizes / 2 * softness) / np.sqrt(2 * np.pi * sizes)
    return centres, sizes[:, None], e / (e.sum(1, keepdims=True) + 1e-7)


# ---- the driver --------------------------------------------------------------------------------------------------------
def cluster_environment(maps, num_clusters: int, softness: float = 5.0, seed: int = 0) -> dict:
    """cluster_dataset.py:64-140 with the pieces above: the largest cluster (stable sort by size, descending) is split,
    label 0 keeping the parent's label and label 1 taking the next counter value."""
    med, mean, count, status = statistics_batch(maps)
    if status.any():
        raise RuntimeError(f"images {np.flatnonzero(status).tolist()} cannot be clustered")
    N = len(med)
    labels = np.zeros(N, np.int64)
    clusters = [(np.arange(N), 0)]
    counter = 0
    while len(clusters) < num_clusters:
        idx, label = clusters.pop(0)
        if len(idx) < 2:
            raise RuntimeError(f"cluster {label} holds one image")
        half, _, _ = kmeans2(med[idx], seed, split=counter)
        counter += 1
        clusters += [(idx[half == 0], label), (idx[half == 1], counter)]
        labels[idx[half == 1]] = counter
        clusters.sort(key=lambda c: len(c[0]), reverse=True)
    centres, sizes, probs = targets(mean, labels, num_clusters, softness)
    return dict(labels=labels, cam_centers=centres, cam_sizes=sizes, gating_probs=probs, medians=med, means=mean,
                counts=count)
