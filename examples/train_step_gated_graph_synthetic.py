"""The reference's training step (code/train_esac.py:105-183) as ONE captured CUDA graph per image that runs, differentiates
and steps only the experts that drew hypotheses, as train_esac.py:143-145 and ensemble.update (expert_ensemble.py:58-68) do.

The step follows train_esac.py's structure:
  1. the gating network and the draw with util.clamp_probs (api.assign_hypotheses_async; its seed a device tensor the
     graph advances), then ExpertGate.arm with the draw's histogram;
  2. the static `prediction` buffer is zeroed and, in region e, expert e's output is copied into prediction[e];
  3. esac_loss_async on `prediction` as a leaf, then loss.backward() (the coordinate and the gating gradients);
  4. in region e, expert e's backward of prediction.grad[e] and its Adam step;
  5. the gating network's Adam step, on every image.
At every replay a kernel reads the histogram and the graph skips the regions of the experts without hypotheses: their
parameters and Adam state, `step` included, stay as they were, which the ungated graph of
examples/train_step_graph_synthetic.py cannot do.  Adam creates its state lazily at its first step; a step captured in a
region that a warm-up skipped would create it inside the region, so every optimiser's state is created before.

    python examples/train_step_gated_graph_synthetic.py --images 5 --experts 6 --maxexperts 2 --check

--check trains an eager twin beside the graph, from the same parameters and Adam state, in the reference's loop:
api.assign_hypotheses with the seed the graph used, the histogram read to the host, only the experts with hypotheses
forward, backward and step.  After every replay the loss, the coordinate gradient, and every parameter and Adam state of
the experts and the gating must be bitwise the twin's, and the experts without hypotheses must be bitwise unchanged.
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

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import esac_b200.api as esac_api  # noqa: E402
from esac_b200.autograd import esac_loss, esac_loss_async  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE, random_shift  # noqa: E402
from esac_b200.gate import ExpertGate  # noqa: E402
from test_step_graph_synthetic import PerImageFocalDataset  # noqa: E402
from train_step_synthetic import TinyExpert, TinyGating  # noqa: E402

SEED0 = 777   # the draw's seed at the first replay; every replay adds 1


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5)
    ap.add_argument("--experts", type=int, default=6)
    ap.add_argument("--hypotheses", "-hyps", type=int, default=256)     # train_esac.py:29
    ap.add_argument("--maxexperts", type=int, default=2, help="util.clamp_probs: draw from the n most likely experts (-1: all)")
    ap.add_argument("--expertselection", action="store_true", help="one expert per image (train_esac.py:133-135)")
    ap.add_argument("--threshold", type=float, default=10)              # :32
    ap.add_argument("--inlieralpha", type=float, default=100)           # :35
    ap.add_argument("--inlierbeta", type=float, default=0.5)            # :38
    ap.add_argument("--maxreprojection", type=float, default=100)       # :41
    ap.add_argument("--weightrot", type=float, default=1.0)
    ap.add_argument("--weighttrans", type=float, default=100.0)
    ap.add_argument("--losscut", type=float, default=100.0)
    ap.add_argument("--check", action="store_true", help="train an eager twin beside the graph and compare, bitwise")
    return ap.parse_args(argv)


def init_adam_state(opt):
    """The state torch.optim.Adam(capturable=True) creates at its first step, created now: zero moments, step 0 on the
    parameter's device."""
    for group in opt.param_groups:
        for p in group["params"]:
            st = opt.state[p]
            if not st:
                st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)


class AlwaysGate:
    """A gate that runs every region: the ungated step of examples/train_step_graph_synthetic.py (the control)."""

    def arm(self, counts):
        pass

    def run(self, i, fn):
        return fn()


class GatedTraining:
    """The models, optimisers and static buffers of the captured step, and the step itself (gate: an ExpertGate, or
    AlwaysGate for the ungated control)."""

    def __init__(self, opt, trainset, gate):
        dev = torch.device("cuda")
        self.opt, self.gate = opt, gate
        E, M = opt.experts, opt.hypotheses
        H, W = trainset.image_hw[0] // OUTPUT_SUBSAMPLE, trainset.image_hw[1] // OUTPUT_SUBSAMPLE
        self.E, self.M, self.H, self.W = E, M, H, W
        torch.manual_seed(0)
        self.experts = [TinyExpert().to(dev) for _ in range(E)]
        self.gating = TinyGating(E).to(dev)
        # one optimiser per expert (expert_ensemble.py:9-37); capturable: the step count lives on the device
        self.opts = [torch.optim.Adam(m.parameters(), lr=1e-5, capturable=True) for m in self.experts]
        self.gating_opt = torch.optim.Adam(self.gating.parameters(), lr=1e-4, capturable=True)
        for o in self.opts + [self.gating_opt]:
            init_adam_state(o)
        # static inputs and outputs of the graph
        self.image = torch.zeros(1, 1, *trainset.image_hw, device=dev)
        self.priors = torch.zeros(E, 3, H, W, device=dev)
        self.shift = torch.zeros(2, dtype=torch.int32, device=dev)   # util.random_shift, train_esac.py:125
        self.camera = torch.zeros(3, device=dev)
        self.gt_pose = torch.eye(4, device=dev)
        self.seed = torch.tensor([SEED0], dtype=torch.int64, device=dev)
        self.e_hyps = torch.zeros(M, dtype=torch.int64, device=dev)
        self.hist = torch.zeros(E, device=dev)
        self.draw_status = torch.zeros((), dtype=torch.int32, device=dev)
        self.status = torch.zeros((), dtype=torch.int32, device=dev)
        self.prediction = torch.zeros(E, 3, H, W, device=dev)
        for e in range(E):
            self.experts[e].see(self.priors[e])

    def params(self):
        return (self.opt.weightrot, self.opt.weighttrans, self.opt.losscut, self.opt.threshold, self.opt.inlieralpha,
                self.opt.inlierbeta, self.opt.maxreprojection, OUTPUT_SUBSAMPLE)

    def step(self):
        E, gate = self.E, self.gate
        gating_log_probs = self.gating(self.image)                                                # train_esac.py:128
        gating_probs = torch.exp(gating_log_probs).detach()[0]
        esac_api.assign_hypotheses_async(gating_probs, self.M, self.seed, self.e_hyps, self.hist,     # :130-140
                                         self.draw_status, maxExperts=self.opt.maxexperts,
                                         expertSelection=self.opt.expertselection)
        self.seed.add_(1)
        gate.arm(self.hist)
        outs = [None] * E
        with torch.no_grad():
            self.prediction.zero_()

        def forward(e):
            outs[e] = self.experts[e](self.image)[0]
            with torch.no_grad():
                self.prediction[e].copy_(outs[e])
        for e in range(E):                                                                         # :143-145
            gate.run(e, lambda e=e: forward(e))
        leaf = self.prediction.detach().requires_grad_()
        self.gating_opt.zero_grad(set_to_none=True)
        loss = esac_loss_async(leaf, gating_log_probs, self.e_hyps, self.gt_pose, self.shift, self.camera, *self.params(),
                               expert_selection=self.opt.expertselection, status=self.status)     # :151-176
        loss.backward()                                                                            # :178-180

        def backward(e):
            self.opts[e].zero_grad(set_to_none=True)
            torch.autograd.backward(outs[e], leaf.grad[e])
            self.opts[e].step()
        for e in range(E):                                                                         # ensemble.update
            gate.run(e, lambda e=e: backward(e))
        self.gating_opt.step()
        return loss.detach(), leaf.grad

    def capture(self):
        """Warm-up on a side stream, capture, and (gated) finalize.  Returns the graph and its loss and gradient."""
        E, H, W, M = self.E, self.H, self.W, self.M
        esac_api.reserve_backward_async(1, E, H, W, M, OUTPUT_SUBSAMPLE)
        side = torch.cuda.Stream()        # warm up torch's kernels off the default stream
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                self.step()
        torch.cuda.current_stream().wait_stream(side)
        gated = isinstance(self.gate, ExpertGate)
        graph = torch.cuda.CUDAGraph(keep_graph=gated)
        with torch.cuda.graph(graph):
            loss, grad = self.step()
        if gated:
            self.gate.finalize(graph)
        self.seed.fill_(SEED0)
        return graph, loss, grad

    def load(self, trainset, i):
        """Writes image i into the static inputs; returns what the eager loop needs."""
        idx, img, focallength, gt, _, _ = trainset[i]
        pp_x, pp_y = img.size(2) / 2, img.size(1) / 2                                             # :110-112
        padX, padY, shifted = random_shift(img[None].cuda(), OUTPUT_SUBSAMPLE / 2)                # :125
        self.image.copy_(shifted)
        self.priors.copy_(trainset.prediction_for(int(idx)))
        self.shift.copy_(torch.tensor([padX, padY], dtype=torch.int32))
        self.camera.copy_(torch.tensor([float(focallength), pp_x, pp_y]))
        self.gt_pose.copy_(gt)
        return padX, padY, float(focallength), pp_x, pp_y


def state_of(opt_):
    return [t for st in opt_.state.values() for t in (st["step"], st["exp_avg"], st["exp_avg_sq"])]


def tensors_of(model, opt_):
    return [p.detach() for p in model.parameters()] + state_of(opt_)


def same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


class EagerTwin:
    """The reference's loop (train_esac.py:105-183) on copies of the graph's models and optimisers."""

    def __init__(self, T: GatedTraining):
        self.T = T
        self.experts = [copy.deepcopy(m) for m in T.experts]
        self.gating = copy.deepcopy(T.gating)
        for e in range(T.E):
            self.experts[e].see(T.priors[e])
        self.opts = []
        for m, o in zip(self.experts, T.opts):
            self.opts.append(torch.optim.Adam(m.parameters(), lr=1e-5, capturable=True))
            self.opts[-1].load_state_dict(copy.deepcopy(o.state_dict()))   # its own moments, not the graph's
        self.gating_opt = torch.optim.Adam(self.gating.parameters(), lr=1e-4, capturable=True)
        self.gating_opt.load_state_dict(copy.deepcopy(T.gating_opt.state_dict()))

    def step(self, i, padX, padY, f, ppx, ppy):
        T = self.T
        opt = T.opt
        gating_log_probs = self.gating(T.image)
        gating_probs = torch.exp(gating_log_probs).detach()
        e_hyps, hist = esac_api.assign_hypotheses(gating_probs, T.M, SEED0 + i, maxExperts=opt.maxexperts,
                                                  expertSelection=opt.expertselection)
        counts = hist[0].cpu()                                                                    # the host read-back
        active = [e for e in range(T.E) if counts[e] > 0]
        prediction = torch.zeros(T.E, 3, T.H, T.W, device="cuda")
        outs = {}
        for e in active:
            outs[e] = self.experts[e](T.image)[0]
            with torch.no_grad():
                prediction[e] = outs[e]
        prediction.requires_grad_()
        self.gating_opt.zero_grad(set_to_none=True)
        loss = esac_loss(prediction, gating_log_probs, e_hyps[0], T.gt_pose, opt.weightrot, opt.weighttrans, opt.losscut,
                         padX, padY, f, ppx, ppy, opt.threshold, opt.inlieralpha, opt.inlierbeta, opt.maxreprojection,
                         OUTPUT_SUBSAMPLE, expert_selection=opt.expertselection)
        loss.backward()
        for e in active:
            self.opts[e].zero_grad(set_to_none=True)
            torch.autograd.backward(outs[e], prediction.grad[e])
            self.opts[e].step()
        self.gating_opt.step()
        return float(loss.detach()), prediction.grad, e_hyps[0], hist[0], active


def main(argv=None):
    opt = parse(argv)
    torch.backends.cudnn.deterministic = True   # the same convolution algorithm eagerly and in the graph
    torch.backends.cudnn.benchmark = False
    random.seed(0)
    trainset = PerImageFocalDataset(num_experts=opt.experts, length=opt.images, hypotheses=opt.hypotheses, seed=3)
    T = GatedTraining(opt, trainset, ExpertGate(opt.experts))
    graph, loss, grad = T.capture()
    twin = EagerTwin(T) if opt.check else None
    esac_api.set_seed(2020)   # resets the eager and the stream-ordered call counters alike

    failures = 0
    losses = []
    t_total = 0.0
    for i in range(len(trainset)):
        cam = T.load(trainset, i)
        before = [tensors_of(m, o) for m, o in zip(T.experts, T.opts)]
        before = [[t.clone() for t in ts] for ts in before]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.replay()
        lo = float(loss)
        t_total += time.perf_counter() - t0
        active = [e for e in range(T.E) if float(T.hist[e]) > 0]
        if int(T.status) != 0 or int(T.draw_status) != 0:
            print(f"image {i}: bad assignment (draw status {int(T.draw_status)}, loss status {int(T.status)})")
            failures += 1
            continue
        losses.append(lo)
        line = f"image {i}: experts trained {active}, loss {lo:.3f}"
        idle_kept = all(same(before[e], tensors_of(T.experts[e], T.opts[e])) for e in range(T.E) if e not in active)
        line += ", idle experts " + ("untouched" if idle_kept else "MOVED")
        failures += not idle_kept
        if twin is not None:
            ref_loss, ref_grad, ref_hyps, ref_hist, ref_active = twin.step(i, *cam)
            ok = (np.float32(ref_loss) == np.float32(lo) and torch.equal(ref_grad, grad) and ref_active == active
                  and torch.equal(ref_hyps, T.e_hyps) and torch.equal(ref_hist, T.hist)
                  and all(same(tensors_of(a, oa), tensors_of(b, ob))
                          for a, oa, b, ob in zip(twin.experts + [twin.gating], twin.opts + [twin.gating_opt],
                                                  T.experts + [T.gating], T.opts + [T.gating_opt])))
            line += ", eager loop: " + ("bitwise equal" if ok else "DIFFERENT")
            failures += not ok
        print(line, flush=True)
    if losses:
        print(f"mean loss {np.mean(losses):.3f}, {1e3 * t_total / len(trainset):.2f} ms per image (replay + loss read-back)")
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
