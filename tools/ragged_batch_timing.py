"""Wall time of a mixed-shape batch three ways, and loss-kernel bandwidth of a ragged batch.

An Aachen-like batch: 8 images, 480-pixel short side at sub-sampling 8 (60 cells) with each image's own aspect ratio, E = 10
experts, M = 256 hypotheses.  forward_batch and backward_batch run it (a) as one ragged call on a list, (b) as one call
per shape group (the only batched option before lists), (c) as a loop of single-image calls.  Then the reprojection and
coordinate losses (with gradient) run on a ragged batch and on a uniform batch with the same number of cells; the
bandwidth counts the algorithmic bytes (24 B per cell for the reprojection loss, 48 B for the coordinate loss).

    python tools/ragged_batch_timing.py [--reps 5]
"""
from __future__ import annotations

import argparse
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

# 480-pixel short side / 8: portrait and landscape at 4:3, 3:2 and 16:9
SHAPES = [(60, 80), (80, 60), (60, 90), (60, 80), (90, 60), (60, 107), (60, 80), (80, 60)]


def card() -> str:
    name = torch.cuda.get_device_name(0)
    try:
        lim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=20).stdout.strip()
    except Exception:
        lim = "unknown"
    return f"{name}, power limit {lim or 'unknown'}"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--E", type=int, default=10)
    ap.add_argument("--M", type=int, default=256)
    a = ap.parse_args()
    print(card())
    scenes = [make_scene(E=a.E, H=h, W=w, M=a.M, sub=8, seed=b, f=500.0 + 10 * b) for b, (h, w) in enumerate(SHAPES)]
    B = len(scenes)
    coords = [torch.from_numpy(s.coords).cuda() for s in scenes]
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    cams = [[getattr(s, k) for s in scenes] for k in ("shiftX", "shiftY", "f", "ppx", "ppy")]
    tail = scenes[0].params[5:]
    groups = {}
    for b, s in enumerate(SHAPES):
        groups.setdefault(s, []).append(b)

    def sel(v, idx):
        return [v[i] for i in idx]

    outs = torch.zeros(B, 4, 4, device="cuda")
    grads = [torch.zeros_like(c) for c in coords]
    fwd = {
        "ragged": lambda: api.forward_batch(coords, assign, outs, *cams, *tail),
        "per shape group": lambda: [api.forward_batch(torch.stack(sel(coords, g)), assign[g], outs[g], *[sel(c, g) for c in cams], *tail)
                                    for g in groups.values()],
        "single calls": lambda: [api.forward(coords[b], assign[b], outs[b], *scenes[b].params) for b in range(B)],
    }
    bwd = {
        "ragged": lambda: api.backward_batch(coords, grads, assign, gts, 1.0, 100.0, 100.0, *cams, *tail),
        "per shape group": lambda: [api.backward_batch(torch.stack(sel(coords, g)), torch.stack(sel(grads, g)), assign[g], gts[g], 1.0,
                                                       100.0, 100.0, *[sel(c, g) for c in cams], *tail) for g in groups.values()],
        "single calls": lambda: [api.backward(coords[b], grads[b], assign[b], gts[b], 1.0, 100.0, 100.0, *scenes[b].params)
                                 for b in range(B)],
    }
    print(f"batch of {B}: shapes {SHAPES}, E={a.E}, M={a.M}, {len(groups)} shape groups")
    for name, table in (("forward_batch", fwd), ("backward_batch", bwd)):
        for k, fn in table.items():
            print(f"  {name:15s} {k:16s} {timed(fn, a.reps):8.2f} ms")
    # loss kernels: 16 ragged maps at full resolution vs 16 uniform maps with the same total cell count
    big = [(480, 640), (640, 480), (480, 720), (480, 854)] * 4
    cells = sum(h * w for h, w in big)
    side = int(round((cells / len(big)) ** 0.5 / 4)) * 4
    uni = [(side, cells // len(big) // side)] * len(big)
    gen = torch.Generator(device="cuda").manual_seed(0)
    for label, shapes in (("ragged", big), ("uniform", uni)):
        n = sum(h * w for h, w in shapes)
        pred = [torch.randn(3, h, w, device="cuda", generator=gen) for h, w in shapes]
        gt = [p + 0.1 * torch.randn_like(p) for p in pred]
        g = [torch.empty_like(p) for p in pred]
        poses = torch.eye(4, device="cuda").repeat(len(shapes), 1, 1)
        api.reproj_loss(pred, poses, 525.0, 0, 0, 10.0, outGradients=g)
        ms_r = np.median([(api.reproj_loss(pred, poses, 525.0, 0, 0, 10.0, outGradients=g), api.last_stats()["ms_score"])[1]
                          for _ in range(a.reps)])
        ms_c = np.median([(api.coord_loss(pred, gt, 100.0, outGradients=g), api.last_stats()["ms_score"])[1] for _ in range(a.reps)])
        print(f"  loss kernels {label:8s} {len(shapes)} maps, {n} cells: reprojection {ms_r * 1e3:.1f} us "
              f"({24 * n / ms_r / 1e9:.2f} TB/s), coordinate {ms_c * 1e3:.1f} us ({48 * n / ms_c / 1e9:.2f} TB/s)")


if __name__ == "__main__":
    main()
