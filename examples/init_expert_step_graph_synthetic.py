"""The expert-initialisation training step of init_expert_step_synthetic.py (code/init_expert.py:102-135) as ONE CUDA graph
per step.

The stand-in expert's forward, the scene-coordinate loss (autograd.coord_loss_async), backward() and
Adam(capturable=True) are captured once; each step then only writes its image, prior and ground-truth coordinates into
the graph's static tensors and calls replay().  random_shift runs eagerly before the copy into the static image (:110;
the loss takes no shift).  As in the eager example the prediction is one cell larger than the ground truth in each
direction, so the loss crops it, and half of the ground-truth cells are empty.  The StepLR schedule (:87, :134) runs
between replays on the optimiser's tensor learning rate.

    python examples/init_expert_step_graph_synthetic.py --iterations 5 --check

--check runs the same steps eagerly on autograd.coord_loss with Adam(capturable=True), from the same initial parameters,
and asserts after every step that the loss and every parameter are bitwise those of the graph.
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import coord_loss, coord_loss_async  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, SyntheticRoomDataset, random_shift  # noqa: E402
from init_expert_step_synthetic import expert_error  # noqa: E402
from ref_expert_step_graph_synthetic import arguments, train  # noqa: E402


def main() -> int:
    args = arguments(cutloss=100, lrssteps=2)                               # init_expert.py:22-38
    dev = torch.device("cuda")
    trainset = SyntheticRoomDataset(num_experts=1, length=max(args.iterations, 1), seed=13, noise=0.05, gt_valid_frac=0.5)
    H, W = trainset.image_hw[0] // OUTPUT_SUBSAMPLE, trainset.image_hw[1] // OUTPUT_SUBSAMPLE
    image = torch.zeros(1, 1, (H + 1) * OUTPUT_SUBSAMPLE, (W + 1) * OUTPUT_SUBSAMPLE, device=dev)   # the graph's static inputs
    prior = torch.zeros(1, 3, H + 1, W + 1, device=dev)
    gt_coords = torch.zeros(1, 3, H, W, device=dev)

    def write(sample):
        idx, img, _, _, coords, _ = sample
        _, _, shifted = random_shift(img.to(dev), OUTPUT_SUBSAMPLE / 2)    # :110
        p = trainset.prediction_for(int(idx))
        image.copy_(F.pad(shifted, (0, OUTPUT_SUBSAMPLE, 0, OUTPUT_SUBSAMPLE)))   # one more cell of image for the larger map
        prior.copy_(F.pad(p + expert_error(int(idx), p.shape), (0, 1, 0, 1), mode="replicate"))
        gt_coords.copy_(coords)
        return (image, prior), ()

    api.reserve_loss_async(1, H + 1, W + 1)
    return train(args, trainset, write, lambda prediction: coord_loss_async(prediction, gt_coords, args.cutloss),
                 lambda prediction: coord_loss(prediction, gt_coords, args.cutloss), dev)


if __name__ == "__main__":
    sys.exit(main())
