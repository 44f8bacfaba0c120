"""A DSAC*-style training step whose pose loss is the best of M: min_h reference_pose_loss(pose_h), eager and as ONE
captured CUDA graph.

Under a winner-take-all loss the hypothesis that carries the loss is often one the node's own softmax gives p < 1e-3.
With the reference's floor (min_prob = 1e-3) that hypothesis would enter the loss with its initial, unrefined pose and its
gradient would be dropped; min_prob = 0 refines and differentiates all M hypotheses.  The stand-in gating and experts of
custom_loss_step_synthetic.py, the hypothesis draw on the device, the node (autograd.esac_hypotheses_async), the loss, the
trainer's REINFORCE gating term, backward() and Adam(capturable=True) are captured once; each image then writes its
inputs into the graph's static tensors and calls replay().

    python examples/best_of_m_step_synthetic.py --steps 4 --check

--check runs the same step eagerly (autograd.esac_hypotheses, min_prob = 0) on the parameters each replay started from and
with the hypotheses it drew, and compares the loss and every parameter's gradient bitwise.
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import esac_b200.api as api  # noqa: E402
from custom_loss_step_synthetic import Nets  # noqa: E402
from esac_b200.autograd import (esac_hypotheses, esac_hypotheses_async, reference_pose_loss,  # noqa: E402
                                reference_pose_loss_async)
from esac_b200.synth import make_scene  # noqa: E402

TAIL = (10.0, 100.0, 0.5, 100.0)  # inlierThreshold, inlierAlpha, inlierBeta, maxReproj
LOSS = (1.0, 100.0, 100.0)        # wLossRot, wLossTrans, lossCut
SUB = 8
FEATS = 16


def step(nets, prior, feats, gt, node, pose_loss, e_hyps=None, M=None):
    """One training step up to backward(): the best-of-M pose loss plus the REINFORCE gating term.  node(prediction, e_hyps)
    -> (scores, poses, contributing) at min_prob = 0; e_hyps None: drawn on the device from the gating distribution.
    Returns (loss, e_hyps, index of the best hypothesis, its softmax probability)."""
    prediction, log_probs = nets(prior, feats)
    E = prediction.shape[0]
    if e_hyps is None:
        e_hyps = torch.multinomial(torch.exp(log_probs.detach()[0]), M, replacement=True)    # train_esac.py:138
    scores, poses, contributing = node(prediction, e_hyps)
    losses = pose_loss(poses, gt, *LOSS)
    loss, best = losses.min(0)
    counts = torch.zeros(E, device=e_hyps.device).scatter_add_(0, e_hyps, torch.ones_like(e_hyps, dtype=torch.float32))
    total = loss + (loss.detach() * counts * log_probs[0]).sum()                               # train_esac.py:171-176
    total.backward()
    return loss.detach(), e_hyps, best, torch.softmax(scores.detach(), 0).index_select(0, best.reshape(1)).squeeze(0)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--hypotheses", type=int, default=64)
    ap.add_argument("--check", action="store_true", help="compare every replay bitwise with the eager step")
    args = ap.parse_args()
    E, M, H, W = args.experts, args.hypotheses, 60, 80
    dev = torch.device("cuda")
    torch.manual_seed(0)
    nets = Nets(E, FEATS).to(dev)
    opt = torch.optim.Adam(nets.parameters(), lr=1e-3, capturable=True)
    api.context().set_option("fixed_seed", 0)
    # static inputs of the graph
    prior = torch.zeros(E, 3, H, W, device=dev)
    feats = torch.zeros(1, FEATS, device=dev)
    gt = torch.eye(4, device=dev)
    shift = torch.zeros(2, dtype=torch.int32, device=dev)
    cam = torch.ones(3, device=dev)

    def node(prediction, e_hyps):
        return esac_hypotheses_async(prediction, e_hyps, shift, cam, *TAIL, SUB, min_prob=0.0)

    def write(k):
        sc = make_scene(E=E, H=H, W=W, M=M, sub=SUB, seed=3000 + k, outlier_frac=0.6, f=500.0 + 25.0 * k,
                        ppx=W * SUB / 2 + k, ppy=H * SUB / 2 - k, shiftX=k % 5 - 2, shiftY=2 - k % 4)
        gen = torch.Generator().manual_seed(k)
        prior.copy_(torch.from_numpy(sc.coords) + 0.01 * torch.randn(sc.coords.shape, generator=gen))
        feats.copy_(torch.randn(1, FEATS, generator=gen))
        gt.copy_(torch.from_numpy(sc.gt_pose))
        shift.copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
        cam.copy_(torch.tensor([sc.f, sc.ppx, sc.ppy]))
        return sc

    api.reserve_backward_async(1, E, H, W, M, SUB)
    write(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up outside the capture (Adam's state, the node's context)
        for _ in range(2):
            opt.zero_grad(set_to_none=True)
            step(nets, prior, feats, gt, node, reference_pose_loss_async, M=M)
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    opt.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, e_hyps, best, p_best = step(nets, prior, feats, gt, node, reference_pose_loss_async, M=M)
        opt.step()
    grads = [p.grad for p in nets.parameters()]   # the graph's gradient buffers
    ref = Nets(E, FEATS).to(dev)
    for k in range(args.steps):
        sc = write(k)
        start = {n: p.detach().clone() for n, p in nets.named_parameters()}
        api.set_seed(21 + k)
        t0 = time.perf_counter()
        graph.replay()
        torch.cuda.synchronize()
        line = (f"step {k}: best-of-{M} loss {loss.item():.3f} (hypothesis {int(best)}, p = {p_best.item():.1e}), "
                f"replay {(time.perf_counter() - t0) * 1e3:.2f} ms")
        if args.check:
            with torch.no_grad():
                for n, p in ref.named_parameters():
                    p.copy_(start[n])
            ref.zero_grad(set_to_none=True)
            params = (sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy) + TAIL + (SUB,)
            api.set_seed(21 + k)
            ref_loss, *_ = step(ref, prior, feats, gt, lambda pr, eh: esac_hypotheses(pr, eh, *params, min_prob=0.0),
                                reference_pose_loss, e_hyps=e_hyps.clone())
            assert loss.item() == ref_loss.item(), f"step {k}: loss {loss.item()} against eager {ref_loss.item()}"
            for (n, p), mine in zip(ref.named_parameters(), grads):
                assert torch.equal(mine, p.grad), f"step {k}: gradient of {n} differs from the eager step"
            line += ", bitwise the eager step (loss and every parameter's gradient)"
        print(line)
    if args.check:
        print("check ok")
    return 0


if __name__ == "__main__":
    sys.exit(main())
