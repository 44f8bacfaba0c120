"""The expert-initialisation training step (code/init_expert.py:102-135) as ONE CUDA graph per step, fed by a
device-resident image set: the graph captures the set's step (image, normalisation, shift, ground truth and the stand-in
prior attached to each image) together with the stand-in expert's forward, the scene-coordinate loss, backward() and
Adam(capturable=True).  The loop is

    dataset.load_plan(plan)                 # once per epoch: the reference loop's draws, one upload
    for g in plan.groups:
        graphs[g].replay()

The set holds seeded uint8 480x640 images (a room set: ToTensor + Normalize with mean 0.4 / std 0.25, no jitter), their
ground-truth maps (half of the cells empty) and a stand-in expert prior per image.

    python examples/init_expert_step_device_data_synthetic.py --iterations 5 --check

--check runs the host-fed step on the same plan beside it, as init_expert_step_graph_synthetic.py's check does: each
step's item is made on the host with torchvision (ToTensor, Normalize, nn.ZeroPad2d with the plan's pads) and trained
eagerly on autograd.coord_loss with Adam(capturable=True), from the same initial parameters; it asserts after every step
that the step's inputs, the loss and every parameter are bitwise those of the host-fed step.
"""
from __future__ import annotations

import argparse
import copy
import random
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
from torchvision import transforms

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import esac_b200.api as api  # noqa: E402
from esac_b200 import data  # noqa: E402
from esac_b200.autograd import coord_loss, coord_loss_async  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE  # noqa: E402
from ref_expert_step_graph_synthetic import StandInExpert  # noqa: E402

IMAGE_HW = (480, 640)


def synthetic_set(n: int, storage: str = "device", seed: int = 17):
    """n seeded uint8 images with ground truth (half of the cells empty) and a stand-in prior per image; returns the
    set's inputs as the host holds them."""
    rng = np.random.default_rng(seed)
    H, W = IMAGE_HW[0] // OUTPUT_SUBSAMPLE, IMAGE_HW[1] // OUTPUT_SUBSAMPLE
    images = [rng.integers(0, 256, IMAGE_HW + (3,), dtype=np.uint8) for _ in range(n)]
    gt = []
    for _ in range(n):
        g = torch.from_numpy(rng.standard_normal((3, H, W)).astype(np.float32) * 2)
        g[:, torch.from_numpy(rng.random((H, W)) < 0.5)] = 0
        gt.append(g)
    prior = torch.stack(gt) + torch.from_numpy(rng.standard_normal((n, 3, H, W)).astype(np.float32) * 0.5)
    poses = np.repeat(np.eye(4, dtype=np.float32)[None], n, 0)
    return dict(images=images, poses=poses, focal=rng.uniform(500, 600, n), scenes=[0] * n, gt=gt,
                attachments={"prior": prior}, storage=storage)


def host_item(inputs, row):
    """The host-fed route of the reference loop for one plan row: the item's image through ToTensor + Normalize
    (room_dataset.py:91-99) and util.random_shift's nn.ZeroPad2d with the row's pads, its prior and ground truth."""
    i = int(row["image"])
    image = transforms.Normalize([data.ROOM_MEAN] * 3, [data.ROOM_STD] * 3)(transforms.ToTensor()(inputs["images"][i]))
    padX, padY = int(row["padX"]), int(row["padY"])
    image = nn.ZeroPad2d((padX, -padX, padY, -padY))(image.unsqueeze(0))
    return image, inputs["attachments"]["prior"][i].unsqueeze(0), inputs["gt"][i].unsqueeze(0)


def capture(model, optimizer, inputs, cut):
    """One training step on static inputs (image, prior, gt) as a CUDA graph; `inputs()` enqueues what feeds them."""
    def step():
        optimizer.zero_grad(set_to_none=False)
        image, prior, gt = inputs()
        loss = coord_loss_async(model(image, prior), gt, cut)
        loss.backward()
        optimizer.step()
        return loss.detach()

    side = torch.cuda.Stream()   # the first step creates Adam's state and the gradient buffers the graph then owns
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    return graph, loss


def arguments():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--learningrate", "-lr", type=float, default=0.0001)
    ap.add_argument("--cutloss", "-cl", type=float, default=100)
    ap.add_argument("--storage", choices=("device", "pinned"), default="device")
    ap.add_argument("--check", action="store_true", help="compare every step bitwise with the host-fed captured step")
    return ap.parse_args()


def main() -> int:
    args = arguments()
    dev = torch.device("cuda")
    random.seed(1)
    torch.manual_seed(1)
    inputs = synthetic_set(args.iterations + 1, args.storage)
    dataset = data.DeviceImageSet(**inputs)
    plan = dataset.plan(data.RoomDraws([len(dataset)], scene=0))      # one epoch of init_expert.py's draws on one scene
    api.reserve_loss_async(1, IMAGE_HW[0] // OUTPUT_SUBSAMPLE, IMAGE_HW[1] // OUTPUT_SUBSAMPLE)
    out = dataset.outputs(0)

    def device_inputs():
        dataset.step(0)
        return out["image"], out["prior"], out["gt_coords"]

    def adam(m):
        return torch.optim.Adam(m.parameters(), lr=torch.tensor(args.learningrate, device=dev), capturable=True)

    model = StandInExpert().to(dev)
    host_model = copy.deepcopy(model)
    # The uncaptured first step of each route takes plan row 0 (the capture runs nothing); replays go on from row 1.
    dataset.load_plan(plan)
    graph, loss = capture(model, adam(model), device_inputs, args.cutloss)
    if args.check:
        host_opt = adam(host_model)

        def host_step(row):
            image, prior, gt = (v.to(dev) for v in host_item(inputs, row))
            host_opt.zero_grad(set_to_none=False)
            want = coord_loss(host_model(image, prior), gt, args.cutloss)
            want.backward()
            host_opt.step()
            return (image, prior, gt), want.detach()

        host_step(plan.rows[0])
        for (n, p), q in zip(model.named_parameters(), host_model.parameters()):
            assert torch.equal(p, q), f"the first step: parameter {n} differs from the host-fed step"
    for iteration, g in enumerate(plan.groups[1:args.iterations + 1]):
        start_time = time.time()
        graph.replay()
        line = "Iteration: %6d, Loss: %.1f, Time: %.2fs" % (iteration, loss.item(), time.time() - start_time)
        assert int(out["status"].item()) == 0, f"iteration {iteration}: data step status {int(out['status'].item())}"
        if args.check:
            items, want = host_step(plan.rows[iteration + 1])
            for name, t, v in zip(("image", "prior", "gt_coords"), (out["image"], out["prior"], out["gt_coords"]), items):
                assert torch.equal(t, v), f"iteration {iteration}: the step's {name} differs from the host-made item"
            assert torch.equal(loss, want), f"iteration {iteration}: loss {loss.item()} against {want.item()}"
            for (n, p), q in zip(model.named_parameters(), host_model.parameters()):
                assert torch.equal(p, q), f"iteration {iteration}: parameter {n} differs from the host-fed step"
            line += ", bitwise the host-fed step (inputs, loss and parameters)"
        print(line, flush=True)
    if args.check:
        print("check ok")
    return 0


if __name__ == "__main__":
    sys.exit(main())
