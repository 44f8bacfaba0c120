"""The expert-initialisation training step (code/init_expert.py:102-135) with its loss block replaced by the fused kernels.

init_expert.py crops prediction and ground truth to a common size, masks out the cells without ground truth and builds
the robust scene-coordinate loss from ~10 torch ops and four boolean-mask indexings per step (each one a host
synchronisation), then lets autograd differentiate them; `esac_b200.autograd.coord_loss` is the same loss and gradient
from two kernels (esac_b200/csrc/coord_loss.cu).  Dataset and network are stand-ins (esac_b200.compat, a 1x1-conv "expert"
whose input is the ground truth plus the errors of an untrained network, 1 cm to 3 km per cell, so cells fall on both sides
of the cut, and whose output is one cell larger than the ground truth in each direction, so the crop has work to do); the
loop itself is the reference's.  With --check every step's loss and gradient are also evaluated with the original op
sequence in float64 (oracle/coord_loss_oracle.py).

    python examples/init_expert_step_synthetic.py --iterations 5 --check
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from esac_b200.autograd import coord_loss  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, SyntheticRoomDataset, random_shift  # noqa: E402


def expert_error(index: int, shape) -> torch.Tensor:
    """Per-cell errors of a stand-in expert early in training: random directions, log-uniform lengths from 1 cm to
    ~3 km (a quarter of them beyond the default cut of 100 m); deterministic per image."""
    g = torch.Generator().manual_seed(1000 + index)
    dirn = torch.randn(shape, generator=g)
    dirn /= dirn.norm(dim=1, keepdim=True)
    length = 10.0 ** (torch.rand((shape[0], 1) + tuple(shape[2:]), generator=g) * 5.5 - 2.0)
    return dirn * length


def check_step(prediction, gt_coords, cut, loss_value):
    """The original op sequence in float64 on the same prediction: loss and d loss / d prediction must agree, and the step
    must exercise the mask and both branches of the robust loss."""
    from oracle.coord_loss_oracle import coord_loss_and_grad
    p, q = prediction.detach().cpu()[0], gt_coords.cpu()[0]
    ref, ref_grad = coord_loss_and_grad(p, q, cut, dtype=torch.float64)
    assert ref > 1.0 and abs(ref - loss_value) <= 1e-6 * ref, (ref, loss_value)
    err = (prediction.grad.cpu()[0].double() - ref_grad).abs().max().item()
    assert err <= 1e-5 * ref_grad.abs().max().item(), err
    h, w = q.shape[1:]
    valid = q.abs().sum(0) != 0
    n = (p[:, :h, :w].double() - q.double()).norm(dim=0)[valid]
    assert (~valid).sum() > 100 and (n <= cut).sum() > 100 and (n > cut).sum() > 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--learningrate", "-lr", type=float, default=0.0001)   # init_expert.py:22
    ap.add_argument("--cutloss", "-cl", type=float, default=100)           # :38
    ap.add_argument("--gt-valid-frac", type=float, default=0.5)             # share of cells with ground truth
    ap.add_argument("--check", action="store_true")
    opt = ap.parse_args()
    dev = torch.device("cuda")
    trainset = SyntheticRoomDataset(num_experts=1, length=max(opt.iterations, 1), seed=13, noise=0.05,
                                    gt_valid_frac=opt.gt_valid_frac)
    trainset_loader = torch.utils.data.DataLoader(trainset, shuffle=False, num_workers=0)
    model = nn.Conv2d(3, 3, 1).to(dev)                                      # stand-in for Expert
    nn.init.eye_(model.weight.view(3, 3))
    nn.init.zeros_(model.bias)
    optimizer = torch.optim.Adam(model.parameters(), lr=opt.learningrate)   # :86
    out = []
    for iteration, (idx, image, focallength, gt_pose, gt_coords, gt_expert) in enumerate(trainset_loader):   # :102
        start_time = time.time()
        gt_coords = gt_coords.to(dev)                                       # :106
        image = image.to(dev)                                               # :107
        padX, padY, image = random_shift(image, OUTPUT_SUBSAMPLE / 2)       # :110 (the loss takes no shift)
        prior = trainset.prediction_for(int(idx))
        prior = F.pad((prior + expert_error(int(idx), prior.shape)).to(dev), (0, 1, 0, 1), mode="replicate")
        prediction = model(prior)                                           # :112, [1,3,61,81] against [1,3,60,80]
        robust_loss = coord_loss(prediction, gt_coords, opt.cutloss)        # :114-130 in one call
        if opt.check:
            prediction.retain_grad()
        robust_loss.backward()                                              # :132
        loss_value = robust_loss.item()
        if opt.check:
            check_step(prediction, gt_coords, opt.cutloss, loss_value)
        optimizer.step()                                                    # :133
        optimizer.zero_grad()                                               # :135
        print("Iteration: %6d, Loss: %.1f, Time: %.2fs" % (iteration, loss_value, time.time() - start_time), flush=True)  # :137
        out.append(loss_value)
    return out


if __name__ == "__main__":
    main()
