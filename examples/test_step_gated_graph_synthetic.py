"""The reference's inference loop (code/test_esac.py:137-230) as ONE captured CUDA graph per image that runs only the experts
that drew hypotheses, as test_esac.py:179-185 does.

The gating network, the hypothesis draw with util.clamp_probs (api.assign_hypotheses_async: clamp + multinomial + histc in
one kernel, its seed a device tensor the graph advances), the experts and esac.forward (api.forward_async) are captured
once.  Each expert runs in a region of an ExpertGate armed with the draw's histogram: at every replay a kernel reads the
histogram and the graph skips the experts without hypotheses, whose planes stay zero (esac.forward never reads them).
The stand-ins and the per-image focal lengths are those of examples/test_step_graph_synthetic.py.

    python examples/test_step_gated_graph_synthetic.py --images 8 --experts 6 --maxexperts 2 --check

--check runs the reference's loop eagerly beside the graph: api.assign_hypotheses with the seed the graph used, the
histogram read to the host, only the experts with hypotheses, zero planes elsewhere, and eager esac.forward.  Every
image's assignment, pose and expert must be bitwise the replay's.  Eager and stream-ordered calls count their seeds
apart, so eager call i after set_seed(s) draws the minimal sets of replay i.
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import esac  # noqa: E402  (this repository's drop-in module)
import esac_b200.api as esac_api  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE  # noqa: E402
from esac_b200.gate import ExpertGate  # noqa: E402
from esac_b200.synth import pose_error  # noqa: E402
from test_step_graph_synthetic import PerImageFocalDataset  # noqa: E402
from train_step_synthetic import TinyExpert, TinyGating  # noqa: E402

SEED0 = 4242   # the draw's seed at the first replay; every replay adds 1


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--experts", type=int, default=6)
    ap.add_argument("--hypotheses", "-hyps", type=int, default=256)     # test_esac.py:29
    ap.add_argument("--maxexperts", type=int, default=2, help="util.clamp_probs: draw from the n most likely experts (-1: all)")
    ap.add_argument("--expertselection", action="store_true", help="one expert per image (test_esac.py:169-171)")
    ap.add_argument("--threshold", type=float, default=10)              # :32
    ap.add_argument("--inlieralpha", type=float, default=100)           # :35
    ap.add_argument("--inlierbeta", type=float, default=0.5)            # :38
    ap.add_argument("--maxreprojection", type=float, default=100)       # :41
    ap.add_argument("--check", action="store_true", help="compare every image with the eager loop, bitwise")
    opt = ap.parse_args(argv)
    torch.backends.cudnn.deterministic = True   # the same convolution algorithm eagerly and in the graph
    torch.backends.cudnn.benchmark = False
    dev = torch.device("cuda")
    E, M = opt.experts, opt.hypotheses
    testset = PerImageFocalDataset(num_experts=E, length=opt.images, hypotheses=M, seed=11, training=False)
    H, W = testset.image_hw[0] // OUTPUT_SUBSAMPLE, testset.image_hw[1] // OUTPUT_SUBSAMPLE
    torch.manual_seed(0)
    experts = [TinyExpert().to(dev).eval() for _ in range(E)]
    gating = TinyGating(E).to(dev).eval()
    thresholds = (opt.threshold, opt.inlieralpha, opt.inlierbeta, opt.maxreprojection, OUTPUT_SUBSAMPLE)

    # static inputs and outputs of the graph
    image = torch.zeros(1, 1, *testset.image_hw, device=dev)
    priors = torch.zeros(E, 3, H, W, device=dev)      # what the stand-in experts "see" in the image
    camera = torch.zeros(3, device=dev)               # focal length, principal point
    shift = torch.zeros(2, dtype=torch.int32, device=dev)   # test_esac.py does not shift at test time
    seed = torch.tensor([SEED0], dtype=torch.int64, device=dev)
    e_hyps = torch.zeros(M, dtype=torch.int64, device=dev)
    hist = torch.zeros(E, device=dev)
    draw_status = torch.zeros((), dtype=torch.int32, device=dev)
    prediction = torch.zeros(E, 3, H, W, device=dev)
    pose = torch.zeros(4, 4, device=dev)
    expert = torch.zeros((), dtype=torch.int64, device=dev)
    status = torch.zeros((), dtype=torch.int32, device=dev)
    for e in range(E):
        experts[e].see(priors[e])
    gate = ExpertGate(E)

    def step():
        with torch.no_grad():
            gating_probs = torch.exp(gating(image))[0]                                         # test_esac.py:163
            esac_api.assign_hypotheses_async(gating_probs, M, seed, e_hyps, hist, draw_status,  # :165-177
                                             maxExperts=opt.maxexperts, expertSelection=opt.expertselection)
            seed.add_(1)
            gate.arm(hist)
            prediction.zero_()
            for e in range(E):                                                                  # :179-185
                gate.run(e, lambda e=e: prediction[e].copy_(experts[e](image)[0]))
        esac_api.forward_async(prediction, e_hyps, shift, camera, *thresholds, pose, expert, status)  # :192-205

    esac_api.reserve_forward_async(1, E, H, W, M, OUTPUT_SUBSAMPLE)
    side = torch.cuda.Stream()            # warm up torch's kernels off the default stream, as torch.cuda.graph expects
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()                            # eagerly: reads the histogram once and runs the experts that drew hypotheses
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        step()
    gate.finalize(graph)                  # each expert's region becomes a conditional node; instantiates the graph
    seed.fill_(SEED0)
    esac_api.set_seed(2020)   # resets the eager and the stream-ordered call counters alike

    failures = 0
    rot_errs, trans_errs = [], []
    t_total = 0.0
    for i in range(len(testset)):
        idx, img, focallength, gt_pose, _, _ = testset[i]
        image.copy_(img[None])
        priors.copy_(testset.prediction_for(int(idx)))
        ppx, ppy = img.size(2) / 2, img.size(1) / 2
        camera.copy_(torch.tensor([float(focallength), ppx, ppy]))                              # :147-150
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.replay()
        out = pose.cpu().numpy()
        t_total += time.perf_counter() - t0
        active = [e for e in range(E) if float(hist[e]) > 0]
        if int(status) != 0 or int(draw_status) != 0:
            print(f"image {i}: bad assignment (draw status {int(draw_status)}, forward status {int(status)})")
            failures += 1
            continue
        rot, trans = pose_error(out, gt_pose.numpy())                                           # :209-222
        rot_errs.append(rot)
        trans_errs.append(trans)
        line = (f"image {i}: f = {float(focallength):7.1f}, experts run {active}, expert {int(expert)}, rot {rot:.3f} deg, "
                f"trans {100 * trans:.2f} cm")
        if opt.check:
            with torch.no_grad():
                gating_probs = torch.exp(gating(image))
                ref_hyps, ref_hist = esac_api.assign_hypotheses(gating_probs, M, SEED0 + i, maxExperts=opt.maxexperts,
                                                                expertSelection=opt.expertselection)
                counts = ref_hist[0].cpu()
                ref_pred = torch.zeros(E, 3, H, W, device=dev)
                for e in range(E):
                    if counts[e] > 0:
                        ref_pred[e] = experts[e](image)[0]
            ref = torch.zeros(4, 4, device=dev)
            ref_e = esac.forward(ref_pred, ref_hyps[0], ref, 0, 0, float(focallength), ppx, ppy, *thresholds)
            same = (torch.equal(ref_hyps[0], e_hyps) and torch.equal(ref_hist[0], hist) and ref_e == int(expert)
                    and np.array_equal(ref.cpu().numpy(), out) and torch.equal(ref_pred, prediction))
            line += ", eager loop: " + ("bitwise equal" if same else "DIFFERENT")
            failures += not same
        print(line, flush=True)
    if rot_errs:
        print(f"median rot {np.median(rot_errs):.3f} deg, median trans {100 * np.median(trans_errs):.2f} cm, "
              f"{1e3 * t_total / len(testset):.2f} ms per image (replay + pose read-back)")
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
