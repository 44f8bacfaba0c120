"""The expert-refinement training step of ref_expert_step_synthetic.py (code/ref_expert.py:95-151) as ONE CUDA graph per step.

The stand-in expert's forward, the reprojection loss (autograd.reproj_loss_async), backward() and Adam(capturable=True) are
captured once; each step then only writes its image, prior, ground truth, pads and camera into the graph's static tensors
and calls replay().  random_shift runs eagerly before the copy into the static image: it pads by host-random amounts, and
those pads reach the loss through a device tensor.  The StepLR schedule (:68, :150) runs between replays on the
optimiser's tensor learning rate, which the graph reads in place.

    python examples/ref_expert_step_graph_synthetic.py --iterations 5 --check

--check runs the same steps eagerly on autograd.reproj_loss with Adam(capturable=True), from the same initial parameters,
and asserts after every step that the loss and every parameter are bitwise those of the graph.
"""
from __future__ import annotations

import argparse
import copy
import sys
import time
from pathlib import Path

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import reproj_loss, reproj_loss_async  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, SyntheticRoomDataset, random_shift  # noqa: E402


class StandInExpert(nn.Module):
    """The 1x1-conv stand-in of the eager examples reduced to its diagonal (a per-channel scale and shift of the prior the
    dataset attaches to each image), plus a learned per-channel weight of the shifted image averaged over 8x8 pixels, so
    that the graph's static image feeds the prediction as the expert's input does.  Elementwise ops and an average pool
    only: their backward sums in the same order in a graph and eagerly, which --check relies on."""

    def __init__(self):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(1, 3, 1, 1))
        self.shift = nn.Parameter(torch.zeros(1, 3, 1, 1))
        self.image_weight = nn.Parameter(torch.zeros(1, 3, 1, 1))

    def forward(self, image, prior):
        return prior * self.scale + self.shift + F.avg_pool2d(image, OUTPUT_SUBSAMPLE) * self.image_weight


def train(args, trainset, write, loss_graph, loss_eager, dev) -> int:
    """The loop both graph examples share.  write(sample) fills the static tensors and returns what loss_eager needs
    besides the prediction; loss_graph(prediction) is the captured loss node.  Iteration 0 runs uncaptured on a side
    stream (it creates Adam's state and the gradient buffers the graph then owns); iterations 1.. are replays."""
    loader = torch.utils.data.DataLoader(trainset, shuffle=False, num_workers=0)
    model = StandInExpert().to(dev)
    ref = copy.deepcopy(model) if args.check else None

    def optimiser(m):
        opt = torch.optim.Adam(m.parameters(), lr=torch.tensor(args.learningrate, device=dev), capturable=True)
        return opt, torch.optim.lr_scheduler.StepLR(opt, step_size=args.lrssteps, gamma=args.lrsgamma)

    optimizer, scheduler = optimiser(model)
    ref_opt, ref_sched = optimiser(ref) if args.check else (None, None)

    def step():
        optimizer.zero_grad(set_to_none=False)
        loss = loss_graph(model(*static_inputs))
        loss.backward()
        optimizer.step()
        return loss.detach()   # no reference to this step's autograd graph outlives it

    graph, out = None, []
    for iteration, sample in enumerate(loader):
        start_time = time.time()
        static_inputs, extra = write(sample)
        if graph is None:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                loss = step()
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                captured = step()
        else:
            graph.replay()
            loss = captured
        scheduler.step()
        loss_value = loss.item()
        line = "Iteration: %6d, Loss: %.1f, Time: %.2fs" % (iteration, loss_value, time.time() - start_time)
        if args.check:
            ref_opt.zero_grad(set_to_none=False)
            want = loss_eager(ref(*static_inputs), *extra)
            want.backward()
            ref_opt.step()
            ref_sched.step()
            assert torch.equal(loss, want.detach()), f"iteration {iteration}: loss {loss_value} against eager {want.item()}"
            for (n, p), q in zip(model.named_parameters(), ref.parameters()):
                assert torch.equal(p, q), f"iteration {iteration}: parameter {n} differs from the eager step"
            line += ", bitwise the eager step (loss and parameters)"
        print(line, flush=True)
        out.append(loss_value)
    if args.check:
        print("check ok")
    return 0


def arguments(cutloss: float, lrssteps: int):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--learningrate", "-lr", type=float, default=0.0001)
    ap.add_argument("--cutloss", "-cl", type=float, default=cutloss)
    # the reference halves the rate every 400 000 steps; a short run halves it every `lrssteps` to show the schedule
    ap.add_argument("--lrssteps", "-lrss", type=int, default=lrssteps)
    ap.add_argument("--lrsgamma", "-lrsg", type=float, default=0.5)
    ap.add_argument("--check", action="store_true", help="compare every step bitwise with the eager step")
    return ap.parse_args()


def main() -> int:
    args = arguments(cutloss=10, lrssteps=2)                                # ref_expert.py:22-37
    dev = torch.device("cuda")
    trainset = SyntheticRoomDataset(num_experts=1, length=max(args.iterations, 1), seed=11, noise=0.05)
    H, W = trainset.image_hw[0] // OUTPUT_SUBSAMPLE, trainset.image_hw[1] // OUTPUT_SUBSAMPLE
    image = torch.zeros(1, 1, *trainset.image_hw, device=dev)               # the graph's static inputs
    prior = torch.zeros(1, 3, H, W, device=dev)
    gt_pose = torch.zeros(1, 4, 4, device=dev)
    shifts = torch.zeros(1, 2, dtype=torch.int32, device=dev)
    cameras = torch.zeros(1, 3, device=dev)
    cx, cy = trainset.image_hw[1] / 2, trainset.image_hw[0] / 2             # the image centre (:118-119)

    def write(sample):
        idx, img, focallength, pose, _, _ = sample
        padX, padY, shifted = random_shift(img.to(dev), OUTPUT_SUBSAMPLE / 2)   # :100, host-random pads
        f = float(focallength[0])                                               # :114
        image.copy_(shifted)
        prior.copy_(trainset.prediction_for(int(idx)))
        gt_pose.copy_(pose)
        shifts.copy_(torch.tensor([[padX, padY]], dtype=torch.int32))
        cameras.copy_(torch.tensor([[f, cx, cy]]))
        return (image, prior), (padX, padY, f)

    api.reserve_loss_async(1, H, W)
    return train(args, trainset, write,
                 lambda prediction: reproj_loss_async(prediction, gt_pose, shifts, cameras, args.cutloss, OUTPUT_SUBSAMPLE),
                 lambda prediction, padX, padY, f: reproj_loss(prediction, gt_pose, f, padX, padY, args.cutloss,
                                                               OUTPUT_SUBSAMPLE, cx, cy),
                 dev)


if __name__ == "__main__":
    sys.exit(main())
