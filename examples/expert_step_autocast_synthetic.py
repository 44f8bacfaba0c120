"""The two expert training steps (init_expert.py:106-132 with the scene-coordinate loss, ref_expert.py:103-150 with the
reprojection loss) of a stand-in FCN run under torch.autocast: bfloat16, and float16 with torch.amp.GradScaler.  The
expert's output is 16-bit (its last layer is a conv, and the scene centre is added in place, as expert.py:83-85 does), and
the loss nodes take it as it is: no prediction.float(), a float32 loss, and 16-bit gradients scaled on the device before
they are rounded.  Each mode runs eagerly (autograd.coord_loss / reproj_loss) and captured in a CUDA graph
(autograd.coord_loss_async / reproj_loss_async): forward, loss and scaled backward in the graph, the scaler's step and
update between replays.

    python examples/expert_step_autocast_synthetic.py --steps 5 --check

--check computes, before every step, the loss and the gradient reaching the prediction along the prediction.float() route
(the float32 node on the upcast output, with the same upstream scale) and asserts that the step's are bitwise the same.
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200 import autograd as ag  # noqa: E402

SUB, H, W, B = 8, 60, 80, 2
F, CX, CY = 525.0, W * SUB / 2, H * SUB / 2


class StandInExpert(nn.Module):
    """Three stride-2 convs from the 480x640 image to 3 x 60 x 80 scene coordinates around the scene centre."""

    def __init__(self, centre):
        super().__init__()
        self.net = nn.Sequential(nn.Conv2d(3, 32, 3, stride=2, padding=1), nn.ReLU(),
                                 nn.Conv2d(32, 32, 3, stride=2, padding=1), nn.ReLU(),
                                 nn.Conv2d(32, 3, 3, stride=2, padding=1))
        self.register_buffer("centre", centre.reshape(1, 3, 1, 1))

    def forward(self, image):
        sc = self.net(image)
        sc.add_(self.centre)   # in place, as expert.py: the output keeps the conv's 16-bit dtype
        return sc


def synthetic_step_data(rng, dev):
    """A batch of images, camera->world ground truths, scene coordinates (10% of cells without ground truth), pads."""
    ys, xs = np.mgrid[0:H, 0:W]
    poses, coords = [], []
    for _ in range(B):
        a = rng.uniform(-0.3, 0.3, 3)
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + K + K @ K / 2
        u, _, vt = np.linalg.svd(R)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = u @ vt, rng.uniform(-1, 1, 3)
        z = rng.uniform(2.0, 5.0, (H, W))
        cam = np.stack([(xs * SUB + SUB / 2 - CX) * z / F, (ys * SUB + SUB / 2 - CY) * z / F, z, np.ones_like(z)])
        world = (T @ cam.reshape(4, -1))[:3].reshape(3, H, W)
        world[:, rng.random((H, W)) < 0.1] = 0.0
        poses.append(T)
        coords.append(world)
    image = torch.from_numpy(rng.standard_normal((B, 3, H * SUB, W * SUB)).astype(np.float32)).to(dev)
    return (image, torch.from_numpy(np.stack(poses).astype(np.float32)).to(dev),
            torch.from_numpy(np.stack(coords).astype(np.float32)).to(dev))


def bitwise(a, b) -> bool:
    """The same bits, NaN matching any NaN."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0).view(torch.int16), b.masked_fill(nb, 0).view(torch.int16))


def run(stage, dtype, graph_mode, args, dev) -> None:
    rng = np.random.default_rng(3)
    torch.manual_seed(0)
    image0, _, coords0 = synthetic_step_data(rng, dev)
    net = StandInExpert(torch.stack([coords0[:, c][coords0[:, c] != 0].mean() for c in range(3)])).to(dev)
    opt = torch.optim.SGD(net.parameters(), lr=1e-6)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16) if dtype == torch.float16 else None
    # the step's inputs live in static tensors (the graph reads them in place)
    image, gt_pose, gt_coords = image0.clone(), torch.zeros(B, 4, 4, device=dev), coords0.clone()
    shifts = torch.zeros(B, 2, dtype=torch.int32, device=dev)
    cameras = torch.tensor([[F, CX, CY]] * B, device=dev)

    def loss_of(p, upcast=False):
        p = p.float() if upcast else p
        if stage == "init":
            return (ag.coord_loss_async if graph_mode else ag.coord_loss)(p, gt_coords, args.cutloss)
        if graph_mode:
            return ag.reproj_loss_async(p, gt_pose, shifts, cameras, args.cutloss, SUB)
        s = shifts.cpu()
        return ag.reproj_loss(p, gt_pose, F, s[:, 0], s[:, 1], args.cutloss, SUB, CX, CY)

    def scaled(loss):
        return scaler.scale(loss) if scaler else loss

    def step():
        """Forward, loss and scaled backward; returns the loss and the prediction's gradient.  No reference to the step's
        autograd graph outlives it (a graph kept alive across the capture would tie the parameters' gradient accumulation
        to another stream)."""
        opt.zero_grad(set_to_none=False)
        with torch.autocast("cuda", dtype=dtype):
            p = net(image)
            p.retain_grad()
            loss = loss_of(p)
        scaled(loss).backward()
        return loss.detach(), p.grad

    def upcast_route():
        """The loss and the prediction's gradient along prediction.float(), on the current parameters and inputs."""
        with torch.autocast("cuda", dtype=dtype):
            p_ref = net(image)
            loss_ref = loss_of(p_ref, upcast=True)
        (g_ref,) = torch.autograd.grad(scaled(loss_ref), p_ref)
        return loss_ref.detach(), g_ref

    graph = None
    for it in range(args.steps):
        img, poses, coords = synthetic_step_data(rng, dev)
        image.copy_(img)
        gt_pose.copy_(poses)
        gt_coords.copy_(coords)
        shifts.copy_(torch.from_numpy(rng.integers(-4, 5, (B, 2)).astype(np.int32)))
        if args.check:
            loss_ref, g_ref = upcast_route()
        if not graph_mode:
            loss, grad = step()
        elif graph is None:   # the first step runs uncaptured on a side stream, then the same step is captured
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                loss, grad = step()
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                captured = step()
        else:
            graph.replay()
            loss, grad = captured
        line = f"{stage} {str(dtype)[6:]:8s} {'graph' if graph_mode else 'eager'} step {it}: loss {loss.item():.4f}"
        if args.check:
            assert loss.dtype == torch.float32 and torch.equal(loss, loss_ref), (loss, loss_ref)
            assert grad.dtype == dtype and bitwise(grad, g_ref), f"{line}: the prediction's gradient differs"
            line += ", loss and prediction gradient bitwise those of prediction.float()"
        if scaler:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        print(line, flush=True)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--cutloss", "-cl", type=float, default=10.0)
    ap.add_argument("--check", action="store_true", help="compare every step with the prediction.float() route")
    args = ap.parse_args()
    dev = torch.device("cuda")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True   # the same conv algorithms in the step and in the check's forward
    api.reserve_loss_async(B, H, W)
    for stage in ("init", "ref"):
        for dtype in (torch.bfloat16, torch.float16):
            for graph_mode in (False, True):
                run(stage, dtype, graph_mode, args, dev)
    if args.check:
        print("check passed")
    return 0


if __name__ == "__main__":
    sys.exit(main())
