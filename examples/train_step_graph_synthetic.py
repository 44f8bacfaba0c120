"""The reference's training step (code/train_esac.py:105-183) as ONE captured CUDA graph per image.

The gating network, the hypothesis draw (torch.multinomial: torch's generator is graph-safe), every expert's network,
esac.backward with the gating gradient (autograd.esac_loss_async), loss.backward() and the Adam steps (capturable=True)
are captured once with torch.cuda.graph; each image then only writes its pixels, its random shift, its focal length and
its ground-truth pose into the graph's static inputs and calls replay().  esac.backward is the stream-ordered
api.backward_async, which reads the seed, the shift, the camera and the ground truth from device memory when it runs and
picks the refinement's CTA groups on the device, so every replay draws fresh minimal sets for its own image.  The
stand-ins are those of examples/train_step_synthetic.py, with a focal length per image as in
examples/test_step_graph_synthetic.py.  Where the graph differs from train_esac.py:
  - every expert runs and steps on every image (a graph is a fixed sequence of kernels; which experts receive hypotheses
    is data-dependent): an expert without hypotheses gets a zero gradient, and Adam still moves it by its momentum;
  - util.clamp_probs is not applied before the draw (it edits the probabilities on the host);
  - the gradients are set by the captured backward instead of being zeroed and accumulated.

    python examples/train_step_graph_synthetic.py --images 8 --check

--check compares every replay's loss and coordinate gradient bitwise with eager esac.backward on the graph's own
coordinates and assignment.  The gradient is copied out by a hook inside the graph.  Eager and stream-ordered calls count
their seeds apart, so the eager calls in between do not disturb the graph's draws.
"""
from __future__ import annotations

import argparse
import random
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import esac  # noqa: E402  (this repository's drop-in module)
import esac_b200.api as esac_api  # noqa: E402
from esac_b200.autograd import esac_loss_async  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, random_shift  # noqa: E402
from test_step_graph_synthetic import PerImageFocalDataset  # noqa: E402
from train_step_synthetic import TinyExpert, TinyGating  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--hypotheses", "-hyps", type=int, default=256)     # train_esac.py:29
    ap.add_argument("--threshold", type=float, default=10)              # :32
    ap.add_argument("--inlieralpha", type=float, default=100)           # :35
    ap.add_argument("--inlierbeta", type=float, default=0.5)            # :38
    ap.add_argument("--maxreprojection", type=float, default=100)       # :41
    ap.add_argument("--weightrot", type=float, default=1.0)
    ap.add_argument("--weighttrans", type=float, default=100.0)
    ap.add_argument("--losscut", type=float, default=100.0)
    ap.add_argument("--check", action="store_true", help="compare every replay with eager esac.backward, bitwise")
    opt = ap.parse_args()
    dev = torch.device("cuda")
    E, M = opt.experts, opt.hypotheses
    trainset = PerImageFocalDataset(num_experts=E, length=opt.images, hypotheses=M, seed=3)
    H, W = trainset.image_hw[0] // OUTPUT_SUBSAMPLE, trainset.image_hw[1] // OUTPUT_SUBSAMPLE
    torch.manual_seed(0)
    random.seed(0)
    experts = [TinyExpert().to(dev) for _ in range(E)]
    gating = TinyGating(E).to(dev)
    # one optimiser per expert (expert_ensemble.py:9-37); capturable: the step count lives on the device
    opts = [torch.optim.Adam(m.parameters(), lr=1e-5, capturable=True) for m in experts]
    opts.append(torch.optim.Adam(gating.parameters(), lr=1e-4, capturable=True))

    # static inputs and outputs of the graph
    image = torch.zeros(1, 1, *trainset.image_hw, device=dev)
    priors = torch.zeros(E, 3, H, W, device=dev)      # what the stand-in experts "see" in the image
    shift = torch.zeros(2, dtype=torch.int32, device=dev)   # util.random_shift, train_esac.py:125
    camera = torch.zeros(3, device=dev)               # focal length, principal point
    gt_pose = torch.eye(4, device=dev)
    status = torch.zeros((), dtype=torch.int32, device=dev)
    grad_copy = torch.zeros(E, 3, H, W, device=dev)   # d loss / d prediction, copied out by a hook in the graph
    for e in range(E):
        experts[e].see(priors[e])

    def keep_gradient(g):
        grad_copy.copy_(g)                # returns nothing: the gradient itself flows on unchanged

    def step():
        gating_log_probs = gating(image)                                                        # train_esac.py:128
        gating_probs = torch.exp(gating_log_probs).detach()
        e_hyps = torch.multinomial(gating_probs[0], M, replacement=True)                        # :138 (no .cpu())
        prediction = torch.stack([experts[e](image)[0] for e in range(E)])                      # :143-145, every expert
        prediction.register_hook(keep_gradient)
        loss = esac_loss_async(prediction, gating_log_probs, e_hyps, gt_pose, shift, camera, opt.weightrot,
                               opt.weighttrans, opt.losscut, opt.threshold, opt.inlieralpha, opt.inlierbeta,
                               opt.maxreprojection, OUTPUT_SUBSAMPLE, status=status)           # :151-176
        loss.backward()                                                                          # :178-180
        for o in opts:                                                                           # ensemble.update
            o.step()
        return loss.detach(), prediction.detach(), e_hyps

    esac_api.reserve_backward_async(1, E, H, W, M, OUTPUT_SUBSAMPLE)
    side = torch.cuda.Stream()            # warm up torch's kernels and Adam's state off the default stream
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            for o in opts:
                o.zero_grad(set_to_none=True)
            step()
    torch.cuda.current_stream().wait_stream(side)
    for o in opts:
        o.zero_grad(set_to_none=True)     # the captured backward allocates the gradients and sets them on every replay
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, prediction, e_hyps = step()
    esac_api.set_seed(2020)   # resets the eager and the stream-ordered call counters alike

    failures = 0
    losses = []
    t_total = 0.0
    for i in range(len(trainset)):
        idx, img, focallength, gt, _, _ = trainset[i]
        pp_x, pp_y = img.size(2) / 2, img.size(1) / 2                                            # :110-112
        padX, padY, shifted = random_shift(img[None].to(dev), OUTPUT_SUBSAMPLE / 2)            # :125
        image.copy_(shifted)
        priors.copy_(trainset.prediction_for(int(idx)))
        shift.copy_(torch.tensor([padX, padY], dtype=torch.int32))
        camera.copy_(torch.tensor([float(focallength), pp_x, pp_y]))
        gt_pose.copy_(gt)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.replay()
        lo = float(loss)
        t_total += time.perf_counter() - t0
        if int(status) != 0:
            print(f"image {i}: bad expert index in the assignment")
            failures += 1
            continue
        losses.append(lo)
        line = f"image {i}: f = {float(focallength):7.1f}, shift ({padX:+d}, {padY:+d}), loss {lo:.3f}"
        if opt.check:
            # eager call i on the graph's own coordinates and assignment draws what replay i drew
            ref = torch.zeros_like(prediction)
            ref_loss = esac.backward(prediction, ref, e_hyps, gt_pose, opt.weightrot, opt.weighttrans, opt.losscut, padX,
                                     padY, float(focallength), pp_x, pp_y, opt.threshold, opt.inlieralpha, opt.inlierbeta,
                                     opt.maxreprojection, OUTPUT_SUBSAMPLE)
            same = np.float32(ref_loss) == np.float32(lo) and torch.equal(ref, grad_copy)
            line += ", eager: " + ("bitwise equal" if same else "DIFFERENT")
            failures += not same
        print(line, flush=True)
    if losses:
        print(f"mean loss {np.mean(losses):.3f}, {1e3 * t_total / len(trainset):.2f} ms per image (replay + loss read-back)")
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
