"""Time the captured gated test step (examples/test_eval_graph_synthetic.py) with its evaluation done two ways:

  (a) host:   after every replay, read the pose, expert, status and histogram back and evaluate on the host with
              synth.pose_error, as examples/test_step_*graph_synthetic.py do: the host cannot enqueue image i+1 before
              image i has finished on the GPU;
  (b) device: PoseEvaluator.update inside the graph, and one read-back (records, table, pose file) after the last image.

Both modes use the same inputs, copied non_blocking from pinned memory before each replay, so they differ only in the
evaluation.  The time is a host clock around the whole loop, which ends in a device synchronisation (the last read-back),
divided by the images.  Three alternating runs per mode and configuration (E = 7 and 19, M = 256, 60x80 maps), after a
warm-up run of each; the card's name and power limit are read in the same process.

    python tools/eval_timing.py --images 512 --json /tmp/eval_timing.json
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "examples"))
from esac_b200.api import reserve_forward_async  # noqa: E402
from esac_b200.synth import pose_error  # noqa: E402
from test_eval_graph_synthetic import GatedTestStep, options  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def run_host(t: GatedTestStep, n: int) -> float:
    t.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        t.load(i)
        t.graph.replay()
        out = t.pose.cpu().numpy()
        int(t.expert), int((t.hist > 0).sum())           # the winner and the experts run, as the examples read them
        if int(t.status) == 0:
            pose_error(out, t.gt(i)[0])
    return (time.perf_counter() - t0) / n


def run_device(t: GatedTestStep, n: int) -> float:
    t.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        t.load(i)
        t.graph.replay()
    t.evaluator.table()
    t.evaluator.pose_lines(t.names[:n])
    return (time.perf_counter() - t0) / n


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=64, help="generated images, cycled through")
    ap.add_argument("--experts", type=int, nargs="+", default=[7, 19])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("eval_timing needs a CUDA device")
    result = {"card": card(), "images": a.images, "distinct": a.distinct, "hypotheses": 256, "map": "60x80", "configs": []}
    print(json.dumps(result["card"]))
    reserve_forward_async(1, max(a.experts), 60, 80, 256, 8)   # one workspace for every configuration's captures
    for E in a.experts:
        opt = options(["--images", str(a.images), "--distinct", str(a.distinct), "--experts", str(E)])
        steps = {"host": GatedTestStep(opt, evaluate=False), "device": GatedTestStep(opt, evaluate=True)}
        fns = {"host": run_host, "device": run_device}
        for mode in steps:
            fns[mode](steps[mode], min(a.images, 64))     # warm-up
        ms = {mode: [] for mode in steps}
        for _ in range(a.runs):
            for mode in steps:
                ms[mode].append(1e3 * fns[mode](steps[mode], a.images))
        cfg = {"E": E, "ms_per_image": ms, "median_ms": {m: sorted(v)[len(v) // 2] for m, v in ms.items()}}
        result["configs"].append(cfg)
        print(json.dumps(cfg), flush=True)
        del steps
        torch.cuda.synchronize()
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(result, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
