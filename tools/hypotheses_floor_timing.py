"""Times the hypotheses node's forward + backward at the reference's probability floor (min_prob = 1e-3) and at 0 (every
hypothesis refined and differentiated), on CUDA tensors (GPU only).  Shapes: 60x80 and 480x640 cells, each with E = 7,
M = 256 and E = 20, M = 1024.  One step is api.hypotheses_forward then api.hypotheses_backward with a random upstream on
every hypothesis, timed with CUDA events around both calls (each ends in a host synchronisation).  Prints the card name
and power limit first, then per shape and floor the median and range of --reps steps and the number of refined jobs.

    python tools/hypotheses_floor_timing.py --reps 10
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import esac_b200.api as api  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

SHAPES = [("60x80 E=7 M=256", dict(E=7, H=60, W=80, M=256, sub=8, seed=1)),
          ("60x80 E=20 M=1024", dict(E=20, H=60, W=80, M=1024, sub=8, seed=1)),
          ("480x640 E=7 M=256", dict(E=7, H=480, W=640, M=256, sub=1, seed=2)),
          ("480x640 E=20 M=1024", dict(E=20, H=480, W=640, M=1024, sub=1, seed=2))]
FLOORS = (1e-3, 0.0)


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = ""
    return q or torch.cuda.get_device_name()


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    print(f"card: {card()}", flush=True)
    api.context().set_option("fixed_seed", 1)
    for name, kw in SHAPES:
        sc = make_scene(**kw)
        coords = torch.from_numpy(sc.coords).cuda()
        assign = torch.from_numpy(sc.assign).cuda()
        M = sc.assign.shape[0]
        rng = np.random.default_rng(0)
        d_scores = torch.from_numpy(rng.standard_normal(M)).cuda()
        d_poses = torch.from_numpy(rng.standard_normal((M, 6))).cuda()
        grads = torch.zeros_like(coords)
        for floor in FLOORS:
            def step():
                api.set_seed(5)
                _, _, _, tape = api.hypotheses_forward(coords, assign, *sc.params, minProb=floor)
                api.hypotheses_backward(tape, coords, grads, d_scores, d_poses)

            t = timed(step, args.reps, args.warmup)
            print(json.dumps({"shape": name, "min_prob": floor, "forward_backward_ms": round(t[0], 3),
                              "range_ms": [round(t[1], 3), round(t[2], 3)], "refined_jobs": api.last_stats()["n_contrib"]}),
                  flush=True)


if __name__ == "__main__":
    main()
