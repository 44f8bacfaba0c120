"""Time an end-to-end training iteration (train_esac.py's step) two ways, as ms per iteration:

  captured    python -m esac_b200.train's replay loop: esac_b200.train.CapturedTrainLoop over a device-resident image
              set, one graph replay per iteration (data step, torch gating, the draw, the gated experts' forward, the
              ESAC loss and backward, the active experts' and the gating network's Adam steps, the record);
  reference   train_esac.py's loop as a user runs it with this library today: the image copied to the device, the
              random shift, the eager torch networks, the gating probabilities read back (.cpu()), the draw on the host
              tensors (api.assign_hypotheses), a Python loop over the experts with hypotheses, esac.backward through the
              `esac` shim on prediction.cpu(), the gradients copied back, autograd.backward and the Adam steps.

Both arms train the same networks (networks.Expert, networks.Gating, seeded Kaiming weights) on 480x640 images (60x80
maps) with M = 256, at E in {7, 19} and -maxe in {-1, 2}, with torch's default TF32 convolutions; the captured arm uses
cuDNN's deterministic algorithms, as the command does.  Every shape is warmed up first; each timed window is K iterations
ending in a device synchronise; the arms alternate, R windows each, and the median, min and max per iteration are
reported.  The card's name and power limit are read in the same process.

    python tools/train_timing.py --iters 20 --reps 5 --json /tmp/train_timing.json
"""
from __future__ import annotations

import argparse
import json
import random
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import esac  # noqa: E402
import esac_b200.api as api  # noqa: E402
from esac_b200 import train  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, random_shift  # noqa: E402
from esac_b200.data import DeviceImageSet, Plan, RoomDraws  # noqa: E402
from esac_b200.networks import Expert, Gating  # noqa: E402
from oracle import expert_oracle as XO  # noqa: E402
from oracle import gating_oracle as GO  # noqa: E402

H, W, M, IMAGES = 480, 640, 256, 8


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def networks(E: int, dev):
    gating = Gating(E, 1).to(dev)
    gating.load_state_dict(GO.kaiming_state_dict(E, E, 1))
    experts = []
    for e in range(E):
        sd = XO.kaiming_state_dict(100 + e, mean=(0.5 * e, 0.0, 2.0))
        experts.append(Expert(sd["mean"]).to(dev))
        experts[-1].load_state_dict(sd)
    return gating, experts


def images():
    rng = np.random.default_rng(0)
    return [(rng.random((H // 8, W // 8, 3)).repeat(8, 0).repeat(8, 1) * 255).astype(np.uint8) for _ in range(IMAGES)]


class Captured:
    def __init__(self, E: int, maxe: int, dev):
        opt = train.options(["-hyps", str(M), "-maxe", str(maxe), "-iter", "1", "--seed", "1"])
        poses = np.tile(np.eye(4, dtype=np.float32), (IMAGES, 1, 1))
        self.ds = DeviceImageSet(images(), poses, [525.0] * IMAGES, [0] * IMAGES)
        gating, experts = networks(E, dev)
        gating_opt, expert_opts = train.optimizers(opt, gating, experts)
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
        self.loop = train.CapturedTrainLoop(opt, self.ds, gating, experts, gating_opt, expert_opts, 100000)
        torch.backends.cudnn.deterministic = False
        random.seed(1)
        torch.manual_seed(1)
        draws = RoomDraws([IMAGES], training=True)        # an epoch of 1000 random images of one scene
        self.plan = train.epoch_plan(self.ds, draws)
        self.nets = (gating, experts)

    def window(self, k: int, start: int) -> float:
        p = Plan(self.plan.rows[start:start + k], self.plan.groups[start:start + k], 1)
        return self.loop.run(p) * 1e3 / k


class Reference:
    def __init__(self, E: int, maxe: int, dev):
        self.E, self.maxe, self.dev = E, maxe, dev
        self.gating, self.experts = networks(E, dev)
        self.gating_opt = torch.optim.Adam(self.gating.parameters(), lr=1e-6)
        self.opts = [torch.optim.Adam(m.parameters(), lr=1e-6) for m in self.experts]
        self.frames = [((torch.from_numpy(a).permute(2, 0, 1).float() / 255 - 0.4) / 0.25)[None] for a in images()]
        self.gt_pose = torch.eye(4)
        self.i = 0

    def step(self):
        E = self.E
        image = self.frames[self.i % len(self.frames)].cuda()
        prediction = torch.zeros((E, 3, H // 8, W // 8)).cuda()
        padX, padY, image = random_shift(image, OUTPUT_SUBSAMPLE / 2)
        log_p = self.gating(image)
        probs = torch.exp(log_p).cpu()
        e_hyps, hist = api.assign_hypotheses(probs, M, 1000 + self.i, maxExperts=self.maxe)
        e_hyps, hist = e_hyps[0], hist[0]
        for e, count in enumerate(hist):
            if count > 0:
                prediction[e] = self.experts[e](image)
        grads = torch.zeros(prediction.size())
        loss = esac.backward(prediction.cpu(), grads, e_hyps, self.gt_pose, 1.0, 100.0, 100.0, padX, padY, 525.0,
                             W / 2, H / 2, 10.0, 100.0, 0.5, 100.0, OUTPUT_SUBSAMPLE)
        g_gating = (loss * hist).unsqueeze(0)
        torch.autograd.backward((prediction, log_p), (grads.cuda(), g_gating.cuda()))
        self.gating_opt.step()
        self.gating_opt.zero_grad()
        for e, o in enumerate(self.opts):
            if hist[e] > 0:
                o.step()
                o.zero_grad()
        self.i += 1

    def window(self, k: int, start: int) -> float:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(k):
            self.step()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / k


def case(E: int, maxe: int, k: int, reps: int, dev) -> dict:
    captured = Captured(E, maxe, dev)
    reference = Reference(E, maxe, dev)
    captured.window(k, 0)                  # warm-up of both arms at this shape
    reference.window(k, 0)
    times = {"captured": [], "reference": []}
    for r in range(reps):                  # alternate the arms
        times["captured"].append(captured.window(k, (r + 1) * k))
        times["reference"].append(reference.window(k, 0))
    row = {"E": E, "maxe": maxe, "H": H, "W": W, "M": M, "iters_per_window": k, "windows": reps}
    for arm, ts in times.items():
        row[f"{arm}_ms"] = round(statistics.median(ts), 2)
        row[f"{arm}_min_ms"], row[f"{arm}_max_ms"] = round(min(ts), 2), round(max(ts), 2)
    row["speedup"] = round(row["reference_ms"] / row["captured_ms"], 2)
    losses, statuses = captured.loop.record(0, (reps + 1) * k)
    row["captured_finite"] = bool(np.isfinite(losses).all() and not statuses.any())
    del captured, reference
    torch.cuda.empty_cache()
    return row


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="iterations per timed window")
    ap.add_argument("--reps", type=int, default=5, help="timed windows per arm")
    ap.add_argument("--json", type=str, default="")
    opt = ap.parse_args(argv)
    if opt.iters * (opt.reps + 1) > 1000:
        ap.error("--iters * (--reps + 1) must fit in one epoch of 1000 iterations")
    dev = torch.device("cuda")
    info = card()
    print(json.dumps(info), flush=True)
    api.reserve_backward_async(1, 19, H // 8, W // 8, M, OUTPUT_SUBSAMPLE)   # the largest case, before the first capture
    rows = []
    for E in (7, 19):
        for maxe in (-1, 2):
            rows.append(case(E, maxe, opt.iters, opt.reps, dev))
            print(json.dumps(rows[-1]), flush=True)
    if opt.json:
        Path(opt.json).parent.mkdir(parents=True, exist_ok=True)
        Path(opt.json).write_text(json.dumps({"card": info, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
