"""The reference's inference loop (code/test_esac.py:137-205) as ONE captured CUDA graph per image, with the experts run by
ExpertStack: the gating network (torch), the hypothesis draw (api.assign_hypotheses_async, its seed a device tensor the
graph advances), every expert with hypotheses in one launch per layer (ExpertStack.forward_async reads the draw's
histogram on the device; the planes of the others are zero) and esac.forward (api.forward_async).  No ExpertGate.

The experts have the reference's Expert architecture with seeded Kaiming weights and the images are synthetic, so the
poses mean nothing; what the example shows is the captured step.

    python examples/test_step_expert_stack_graph_synthetic.py --images 4 --experts 5 --check

--check compares every replay with the eager reference loop: api.assign_hypotheses with the seed the graph used, and the
per-expert torch forward (cuDNN, TF32) of the experts with hypotheses.  The histogram must be bitwise the replay's, the
planes of experts without hypotheses exactly zero, and each active expert's prediction within 2e-2 relative error of
the torch loop's (both are TF32; the float64 bar of tests/test_gpu_experts.py holds the two to the exact result).
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as esac_api  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE  # noqa: E402
from esac_b200.experts import ExpertStack, prediction_size  # noqa: E402
from oracle import expert_oracle  # noqa: E402  (seeded Kaiming experts and the torch route of --check)

SEED0 = 777   # the draw's seed at the first replay; every replay adds 1


class TinyGating(torch.nn.Module):
    """A stand-in for the reference's Gating: pooled colour statistics to E log-probabilities."""

    def __init__(self, E):
        super().__init__()
        self.fc = torch.nn.Linear(12, E)

    def forward(self, x):
        return F.log_softmax(self.fc(F.adaptive_avg_pool2d(x, 2).flatten(1)), 1)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--experts", type=int, default=5)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--hypotheses", "-hyps", type=int, default=256)     # test_esac.py:29
    ap.add_argument("--maxexperts", type=int, default=2, help="util.clamp_probs: draw from the n most likely experts (-1: all)")
    ap.add_argument("--check", action="store_true", help="compare every replay with the eager per-expert torch loop")
    opt = ap.parse_args(argv)
    dev = torch.device("cuda")
    E, M, H, W = opt.experts, opt.hypotheses, opt.height, opt.width
    h, w = prediction_size(H, W)
    torch.manual_seed(0)
    sds = [expert_oracle.kaiming_state_dict(10 + e, mean=(float(e), 0.0, 2.0)) for e in range(E)]
    stack = ExpertStack(sds, dev)
    gating = TinyGating(E).to(dev).eval()
    thresholds = (10.0, 100.0, 0.5, 100.0, OUTPUT_SUBSAMPLE)          # test_esac.py:32-41

    image = torch.zeros(1, 3, H, W, device=dev)
    camera = torch.tensor([525.0, W / 2, H / 2], device=dev)
    shift = torch.zeros(2, dtype=torch.int32, device=dev)
    seed = torch.tensor([SEED0], dtype=torch.int64, device=dev)
    e_hyps = torch.zeros(M, dtype=torch.int64, device=dev)
    hist = torch.zeros(1, E, device=dev)
    draw_status = torch.zeros((), dtype=torch.int32, device=dev)
    prediction = torch.zeros(1, E, 3, h, w, device=dev)
    pose = torch.zeros(4, 4, device=dev)
    expert = torch.zeros((), dtype=torch.int64, device=dev)
    status = torch.zeros((), dtype=torch.int32, device=dev)

    def step():
        with torch.no_grad():
            gating_probs = torch.exp(gating(image))[0]                                          # test_esac.py:163
            esac_api.assign_hypotheses_async(gating_probs, M, seed, e_hyps, hist[0], draw_status,  # :165-177
                                             maxExperts=opt.maxexperts)
            seed.add_(1)
            stack.forward_async(image, hist, prediction)                                         # :179-185
        esac_api.forward_async(prediction[0], e_hyps, shift, camera, *thresholds, pose, expert, status)  # :192-205

    stack.reserve(1, H, W)
    esac_api.reserve_forward_async(1, E, h, w, M, OUTPUT_SUBSAMPLE)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    seed.fill_(SEED0)

    failures = 0
    gen = torch.Generator().manual_seed(5)
    for i in range(opt.images):
        low = torch.rand((1, 3, H // 16, W // 16), generator=gen)
        img = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)
        image.copy_((img - 0.4) / 0.25)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.replay()
        torch.cuda.synchronize()
        ms = 1e3 * (time.perf_counter() - t0)
        active = [e for e in range(E) if float(hist[0, e]) > 0]
        line = f"image {i}: experts run {active}, expert {int(expert)}, status {int(status)}, replay {ms:.2f} ms"
        if opt.check:
            with torch.no_grad():
                _, ref_hist = esac_api.assign_hypotheses(torch.exp(gating(image)), M, SEED0 + i,
                                                         maxExperts=opt.maxexperts)
                ok = torch.equal(ref_hist[0].to(dev), hist[0])
                worst = 0.0
                for e in range(E):
                    if float(ref_hist[0, e]) > 0:
                        prev = torch.backends.cudnn.allow_tf32
                        torch.backends.cudnn.allow_tf32 = True
                        ref = expert_oracle.apply(image, {k: v.to(dev) for k, v in sds[e].items()})[0]
                        torch.backends.cudnn.allow_tf32 = prev
                        worst = max(worst, float((prediction[0, e] - ref).norm() / ref.norm()))
                    else:
                        ok = ok and not prediction[0, e].any()
            ok = ok and worst <= 2e-2
            line += f", eager loop: largest relative difference {worst:.2e} " + ("ok" if ok else "DIFFERENT")
            failures += not ok
        print(line, flush=True)
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
