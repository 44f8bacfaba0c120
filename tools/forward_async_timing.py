"""Eager esac.forward against the stream-ordered forward, uncaptured and as CUDA-graph replays (GPU only).

For every shape, R images end in ONE torch.cuda.synchronize():
  eager   esac.forward on CUDA tensors (it synchronises inside every call),
  async   api.forward_async in a loop, uncaptured,
  graph   replays of one captured api.forward_async.
Reported per image: host wall time over the R images, and device time between CUDA events around them.  Shapes: the
reference's native 60x80 maps (sub 8) at (E, M) = (1, 64), (7, 256), (19, 256), (20, 1024), and full 480x640 maps (sub 1)
with E = 7, M = 256.

    python tools/forward_async_timing.py [--images 50] [--json out.json]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import esac_b200.api as api  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

SHAPES = [("60x80 sub 8, E=1 M=64", dict(E=1, H=60, W=80, M=64, sub=8)),
          ("60x80 sub 8, E=7 M=256", dict(E=7, H=60, W=80, M=256, sub=8)),
          ("60x80 sub 8, E=19 M=256", dict(E=19, H=60, W=80, M=256, sub=8)),
          ("60x80 sub 8, E=20 M=1024", dict(E=20, H=60, W=80, M=1024, sub=8)),
          ("480x640 sub 1, E=7 M=256", dict(E=7, H=480, W=640, M=256, sub=1))]
TAIL = (10.0, 100.0, 0.5, 100.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, R):
    """(host ms per image, device ms per image) of R calls of fn ending in one synchronise."""
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(R):
        fn()
    b.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / R
    return wall, a.elapsed_time(b) / R


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", "-R", type=int, default=50)
    ap.add_argument("--json", help="also write the table here")
    opt = ap.parse_args()
    R = opt.images
    name = card()
    print(f"card: {name}", flush=True)
    rows = []
    for _, kw in SHAPES:   # every shape before the first capture: a captured workspace never grows
        api.reserve_forward_async(1, kw["E"], kw["H"], kw["W"], kw["M"], kw["sub"])
    for label, kw in SHAPES:
        sc = make_scene(seed=7, **kw)
        E, H, W, M, sub = kw["E"], kw["H"], kw["W"], kw["M"], kw["sub"]
        coords = torch.from_numpy(sc.coords).cuda()
        assign = torch.from_numpy(sc.assign).cuda()
        out = torch.zeros(4, 4, device="cuda")
        shifts = torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda")
        cams = torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda")
        pose, expert = torch.zeros(4, 4, device="cuda"), torch.zeros((), dtype=torch.int64, device="cuda")
        status = torch.zeros((), dtype=torch.int32, device="cuda")

        def eager():
            api.forward(coords, assign, out, *sc.params)

        def stream_ordered():
            api.forward_async(coords, assign, shifts, cams, *TAIL, sub, pose, expert, status)

        for _ in range(3):
            eager()
            stream_ordered()
        launches = api.last_stats()["kernel_launches"]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            stream_ordered()
        g.replay()
        res = {"shape": label, "kernel_launches": launches}
        for kind, fn in (("eager", eager), ("async", stream_ordered), ("graph", g.replay)):
            res[kind] = timed(fn, R)
        torch.cuda.synchronize()
        assert int(status) == 0
        rows.append(res)
        print(f"{label:26s} launches {launches:4d} | host ms/image: eager {res['eager'][0]:7.3f} async {res['async'][0]:7.3f} "
              f"graph {res['graph'][0]:7.3f} | device ms/image: eager {res['eager'][1]:7.3f} async {res['async'][1]:7.3f} "
              f"graph {res['graph'][1]:7.3f}", flush=True)
        del g
    if opt.json:
        Path(opt.json).write_text(json.dumps({"card": name, "images": R, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
