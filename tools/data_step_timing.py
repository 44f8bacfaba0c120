"""Per-step wall time of the captured expert-initialisation step fed from the host against the same step fed by a
device-resident image set (esac_b200.data), at 480x640, with the set in device memory and in mapped pinned host memory.

Host-fed (INTEGRATION.md's captured init_expert.py loop): a DataLoader(shuffle=True, num_workers=--workers) whose dataset
makes each item's image with ToTensor + Normalize from in-memory uint8 images (no decode: both routes start from decoded,
resized images), the copy to the device, util.random_shift there, the small camera / shift tensors, copy_ into the
graph's static tensors and replay().  Device-fed: one replay of a graph that captures the set's step with the training
step.  Both run the stand-in expert of examples/init_expert_step_device_data_synthetic.py.  Each window is timed with the
host clock between two device synchronisations after --warmup steps.  Prints one JSON line, with the card's name and power
limit read in the same run.

    python tools/data_step_timing.py --steps 200 --warmup 20
"""
from __future__ import annotations

import argparse
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch
from torchvision import transforms

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "examples"))
import esac_b200.api as api  # noqa: E402
from esac_b200 import data  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, random_shift  # noqa: E402
from init_expert_step_device_data_synthetic import IMAGE_HW, capture, synthetic_set  # noqa: E402
from ref_expert_step_graph_synthetic import StandInExpert  # noqa: E402


class HostItems(torch.utils.data.Dataset):
    """The host side of a room dataset item from decoded, resized images: ToTensor + Normalize, ground truth, prior."""

    def __init__(self, inputs):
        self.inputs = inputs
        self.transform = transforms.Compose([transforms.ToTensor(), transforms.Normalize([data.ROOM_MEAN] * 3, [data.ROOM_STD] * 3)])

    def __len__(self):
        return len(self.inputs["images"])

    def __getitem__(self, i):
        return (i, self.transform(self.inputs["images"][i]), float(self.inputs["focal"][i]), self.inputs["gt"][i],
                self.inputs["attachments"]["prior"][i])


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = r.stdout.strip().splitlines()[0].partition(",") if r.returncode == 0 and r.stdout.strip() else ("", "", "")
    return {"gpu": name.strip() or torch.cuda.get_device_name(), "power_limit": power.strip() or "unknown"}


def host_fed(inputs, args, dev):
    model = StandInExpert().to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device=dev), capturable=True)
    static = [torch.zeros(1, 3, *IMAGE_HW, device=dev), torch.zeros(1, *inputs["attachments"]["prior"].shape[1:], device=dev),
              torch.zeros(1, *inputs["gt"][0].shape, device=dev)]
    shifts, cameras = torch.zeros(1, 2, dtype=torch.int32, device=dev), torch.zeros(1, 3, device=dev)
    graph, _ = capture(model, opt, lambda: static, args.cutloss)
    loader = torch.utils.data.DataLoader(HostItems(inputs), shuffle=True, num_workers=args.workers, persistent_workers=args.workers > 0)

    def items():
        while True:
            yield from loader

    it = items()

    def step():
        idx, image, focal, gt, prior = next(it)
        padX, padY, image = random_shift(image.to(dev), OUTPUT_SUBSAMPLE / 2)
        shifts.copy_(torch.tensor([[padX, padY]], dtype=torch.int32))
        cameras.copy_(torch.tensor([[float(focal[0]), IMAGE_HW[1] / 2, IMAGE_HW[0] / 2]]))
        static[0].copy_(image)
        static[1].copy_(prior)
        static[2].copy_(gt)
        graph.replay()

    return timed(step, args)


def device_fed(inputs, storage, args, dev):
    dataset = data.DeviceImageSet(**dict(inputs, storage=storage))
    plan = dataset.plan(data.RoomDraws([len(dataset)]))          # 1000 steps of random images
    out = dataset.outputs(0)
    model = StandInExpert().to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device=dev), capturable=True)
    dataset.load_plan(plan)

    def feed():
        dataset.step(0)
        return out["image"], out["prior"], out["gt_coords"]

    graph, _ = capture(model, opt, feed, args.cutloss)
    dataset.load_plan(plan)
    state = {"step": 0}

    def step():
        if state["step"] == len(plan.groups):
            dataset.load_plan(plan)
            state["step"] = 0
        graph.replay()
        state["step"] += 1

    ms = timed(step, args)
    assert int(out["status"].item()) == 0
    return ms


def timed(step, args) -> float:
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / args.steps * 1e3


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--workers", type=int, default=6, help="DataLoader workers of the host-fed route (the reference's 6)")
    ap.add_argument("--cutloss", type=float, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("data_step_timing needs a CUDA device")
    dev = torch.device("cuda")
    random.seed(0)
    torch.manual_seed(0)
    inputs = synthetic_set(args.images)
    api.reserve_loss_async(1, IMAGE_HW[0] // OUTPUT_SUBSAMPLE, IMAGE_HW[1] // OUTPUT_SUBSAMPLE)
    result = {"what": "captured init_expert step, ms per step", "image": list(IMAGE_HW), "steps": args.steps,
              "warmup": args.warmup, "workers": args.workers, **card()}
    result["host_fed_ms"] = host_fed(inputs, args, dev)
    for storage in ("device", "pinned"):
        result[f"device_fed_{storage}_ms"] = device_fed(inputs, storage, args, dev)
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
