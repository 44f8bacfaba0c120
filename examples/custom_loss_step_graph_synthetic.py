"""The DSAC* training step of custom_loss_step_synthetic.py as ONE captured CUDA graph.

The stand-in gating and experts, the hypothesis draw (torch.multinomial on the device: torch's generator is graph-safe),
the hypotheses node (autograd.esac_hypotheses_async), DSAC*'s `max(angle in degrees, translation error in cm)` loss, the
trainer's REINFORCE gating term (d/d log_probs = loss * histogram(e_hyps), the histogram built on the device with
scatter_add_ as autograd._gating_grad builds it), backward() and Adam(capturable=True) are captured once; each image then
only writes its scene-coordinate prior, features, ground truth, shift and camera into the graph's static inputs and calls
replay().  The node is the stream-ordered hypotheses forward and backward: the seed, shift and camera are read on the device
when the kernels run, and the refinement's CTA groups are picked there, so every replay draws fresh minimal sets.

    python examples/custom_loss_step_graph_synthetic.py --images 4 --check

--check compares every replay bitwise with the same step run eagerly on esac_hypotheses, on the parameters the replay
started from and with the hypotheses the replay drew: the loss and every parameter's gradient.  set_seed before a replay
and before its eager twin makes both draw call 0 of the same seed (eager and stream-ordered calls count apart).
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
from custom_loss_step_synthetic import Nets, dsac_star_loss  # noqa: E402
from esac_b200.autograd import esac_hypotheses, esac_hypotheses_async, pose_to_transform  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

TAIL = (10.0, 100.0, 0.5, 100.0)  # inlierThreshold, inlierAlpha, inlierBeta, maxReproj
SUB = 8
FEATS = 16


def step(nets, prior, feats, gt, node, e_hyps=None, M=None):
    """One training step up to backward(): the expected DSAC* loss plus the REINFORCE gating term.  node(prediction,
    e_hyps) -> (scores, poses, contributing); e_hyps None: drawn on the device from the gating distribution."""
    prediction, log_probs = nets(prior, feats)
    E = prediction.shape[0]
    if e_hyps is None:
        e_hyps = torch.multinomial(torch.exp(log_probs.detach()[0]), M, replacement=True)    # train_esac.py:138
    scores, poses, _ = node(prediction, e_hyps)
    loss = (torch.softmax(scores, 0) * dsac_star_loss(pose_to_transform(poses), gt.double())).sum()
    counts = torch.zeros(E, device=e_hyps.device).scatter_add_(0, e_hyps, torch.ones_like(e_hyps, dtype=torch.float32))
    total = loss + (loss.detach() * counts * log_probs[0]).sum()                               # train_esac.py:171-176
    total.backward()
    return loss.detach(), e_hyps


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4)
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
        return esac_hypotheses_async(prediction, e_hyps, shift, cam, *TAIL, SUB)

    def write(k):
        sc = make_scene(E=E, H=H, W=W, M=M, sub=SUB, seed=2000 + k, outlier_frac=0.6, f=500.0 + 25.0 * k,
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
    with torch.cuda.stream(side):   # warm-up outside the capture (Adam's state, cuBLAS handles, the node's context)
        for _ in range(2):
            opt.zero_grad(set_to_none=True)
            step(nets, prior, feats, gt, node, M=M)
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    opt.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, e_hyps = step(nets, prior, feats, gt, node, M=M)
        opt.step()
    grads = [p.grad for p in nets.parameters()]   # the graph's gradient buffers
    ref = Nets(E, FEATS).to(dev)
    for k in range(args.images):
        sc = write(k)
        start = {n: p.detach().clone() for n, p in nets.named_parameters()}
        api.set_seed(11 + k)
        t0 = time.perf_counter()
        graph.replay()
        torch.cuda.synchronize()
        line = f"image {k}: expected DSAC* loss {loss.item():.3f}, replay {(time.perf_counter() - t0) * 1e3:.2f} ms"
        if args.check:
            with torch.no_grad():
                for n, p in ref.named_parameters():
                    p.copy_(start[n])
            ref.zero_grad(set_to_none=True)
            params = (sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy) + TAIL + (SUB,)
            api.set_seed(11 + k)
            ref_loss, _ = step(ref, prior, feats, gt, lambda pr, eh: esac_hypotheses(pr, eh, *params), e_hyps=e_hyps.clone())
            assert loss.item() == ref_loss.item(), f"image {k}: loss {loss.item()} against eager {ref_loss.item()}"
            for (n, p), mine in zip(ref.named_parameters(), grads):
                assert torch.equal(mine, p.grad), f"image {k}: gradient of {n} differs from the eager step"
            line += ", bitwise the eager step (loss and every parameter's gradient)"
        print(line)
    if args.check:
        print("check ok")
    return 0


if __name__ == "__main__":
    sys.exit(main())
