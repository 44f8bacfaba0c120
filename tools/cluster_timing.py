"""Times clustering a Dubrovnik-sized environment (about 6 000 ragged ground-truth maps, 60x80 and 80x60) two ways, with
the statistics and the hierarchy reported apart:

* device: api.cluster_statistics over the maps in pinned host memory, then cluster_environment's hierarchy (a kmeans2 launch
  and one label read-back per split) and cluster_targets;
* reference route: cluster_dataset.py's per-image torch mask / median / sum on the host, then the hierarchy with
  cv2.kmeans(points, 2, None, (EPS + MAX_ITER, 100, 0.1), 10, KMEANS_PP_CENTERS) (needs cv2; skipped without it).

The maps are generated in memory (SyntheticClusterDataset), so neither side includes file I/O, which the reference's
three loads of every map add on top.  Prints one JSON line per K with the GPU's name and power limit.

    python tools/cluster_timing.py --images 6000 --clusters 10 20 50
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200.cluster import hierarchy  # noqa: E402
from esac_b200.compat import SyntheticClusterDataset  # noqa: E402


def gpu_name_power():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def device_route(maps, K, seed=0):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    med, mean, count, status = api.cluster_statistics(maps)
    med, mean = med.cuda(), mean.cuda()
    torch.cuda.synchronize()
    t1 = time.perf_counter()

    def split(idx, s):
        half, _, _ = api.kmeans2(med[torch.from_numpy(idx).cuda()].contiguous(), seed, split=s)
        return half.cpu().numpy()

    labels = torch.from_numpy(hierarchy(len(maps), K, split)).cuda()
    api.cluster_targets(mean, labels, K)
    torch.cuda.synchronize()
    return t1 - t0, time.perf_counter() - t1


def reference_route(maps, K):
    import cv2
    t0 = time.perf_counter()
    medians = torch.zeros(len(maps), 3)
    for i, m in enumerate(maps):
        d = m.view(3, -1)
        mask = d.sum(0) != 0
        d = d[:, mask]
        medians[i] = d.median(1)[0]
        _ = d.sum(1) / mask.sum()
    pts = medians.numpy()
    t1 = time.perf_counter()
    criteria = (cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 100, 0.1)
    clusters = [pts]
    while len(clusters) < K:
        p = clusters.pop(0)
        _, half, _ = cv2.kmeans(p, 2, None, criteria, 10, cv2.KMEANS_PP_CENTERS)
        clusters += [p[half[:, 0] == 0], p[half[:, 0] == 1]]
        clusters.sort(key=lambda c: c.shape[0], reverse=True)
    return t1 - t0, time.perf_counter() - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=6000)
    ap.add_argument("--clusters", type=int, nargs="+", default=[10, 20, 50])
    ap.add_argument("--repeats", type=int, default=3)
    opt = ap.parse_args()
    ds = SyntheticClusterDataset(length=opt.images, training=False)
    maps = [ds.init_map(i).pin_memory() for i in range(opt.images)]
    device_route(maps[:64], 2)                                   # module load, first launches
    card = gpu_name_power()
    for K in opt.clusters:
        dev, ref = [], []
        for _ in range(opt.repeats):
            dev.append(device_route(maps, K))
            try:
                ref.append(reference_route(maps, K))
            except ImportError:
                pass
        row = {"K": K, "images": opt.images, "gpu": card,
               "device_stats_s": min(d[0] for d in dev), "device_hierarchy_s": min(d[1] for d in dev)}
        if ref:
            row.update(reference_stats_s=min(r[0] for r in ref), reference_hierarchy_s=min(r[1] for r in ref))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
