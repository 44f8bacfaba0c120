"""The reference's inference loop (code/test_esac.py:137-230) as ONE captured CUDA graph per image.

The gating network, the hypothesis draw (torch.multinomial: torch's generator is graph-safe), every expert's network and
esac.forward are captured once with torch.cuda.graph; each image then only writes its pixels and camera into the graph's
static inputs and calls replay().  esac.forward is the stream-ordered api.forward_async, which reads the seed, the shift
and the camera from device memory when it runs, so every replay draws fresh minimal sets and uses the image's own focal
length.  The stand-ins are those of examples/train_step_synthetic.py, on esac_b200.compat.SyntheticRoomDataset with a
focal length per image (as 19Scenes, Aachen and Dubrovnik have).  Unlike test_esac.py, every expert runs on every image:
which experts receive hypotheses is data-dependent, and a graph is a fixed sequence of kernels.

    python examples/test_step_graph_synthetic.py --images 8 --check

--check compares every image's pose and expert bitwise with eager esac.forward on the graph's own coordinates and
assignment.  Eager and stream-ordered calls count their seeds apart, so the eager calls in between do not disturb the
graph's draws.
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
from esac_b200.compat import OUTPUT_SUBSAMPLE, SyntheticRoomDataset  # noqa: E402
from esac_b200.synth import make_scene, pose_error  # noqa: E402
from train_step_synthetic import TinyExpert, TinyGating  # noqa: E402

FOCALS = (525.0, 585.0, 744.4, 1080.0)   # one calibration per image, cycling


class PerImageFocalDataset(SyntheticRoomDataset):
    """SyntheticRoomDataset whose image i is taken with focal length FOCALS[i % 4] (its map is generated through that
    camera, so a pose estimated with another focal length misses the ground truth)."""

    def scene(self, index: int):
        if index not in self._cache:
            H, W = self.image_hw[0] // OUTPUT_SUBSAMPLE, self.image_hw[1] // OUTPUT_SUBSAMPLE
            self._cache[index] = make_scene(E=self.num_experts, H=H, W=W, M=self.hypotheses, sub=OUTPUT_SUBSAMPLE,
                                            seed=self.seed * 100003 + index, outlier_frac=self.outlier_frac, noise=self.noise,
                                            active_only=False, f=FOCALS[index % len(FOCALS)])
        return self._cache[index]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--hypotheses", "-hyps", type=int, default=256)     # test_esac.py:29
    ap.add_argument("--threshold", type=float, default=10)              # :32
    ap.add_argument("--inlieralpha", type=float, default=100)           # :35
    ap.add_argument("--inlierbeta", type=float, default=0.5)            # :38
    ap.add_argument("--maxreprojection", type=float, default=100)       # :41
    ap.add_argument("--check", action="store_true", help="compare every image with eager esac.forward, bitwise")
    opt = ap.parse_args()
    dev = torch.device("cuda")
    E, M = opt.experts, opt.hypotheses
    testset = PerImageFocalDataset(num_experts=E, length=opt.images, hypotheses=M, seed=11, training=False)
    H, W = testset.image_hw[0] // OUTPUT_SUBSAMPLE, testset.image_hw[1] // OUTPUT_SUBSAMPLE
    torch.manual_seed(0)
    experts = [TinyExpert().to(dev).eval() for _ in range(E)]
    gating = TinyGating(E).to(dev).eval()

    # static inputs and outputs of the graph
    image = torch.zeros(1, 1, *testset.image_hw, device=dev)
    priors = torch.zeros(E, 3, H, W, device=dev)      # what the stand-in experts "see" in the image
    camera = torch.zeros(3, device=dev)               # focal length, principal point
    shift = torch.zeros(2, dtype=torch.int32, device=dev)   # test_esac.py does not shift at test time
    pose = torch.zeros(4, 4, device=dev)
    expert = torch.zeros((), dtype=torch.int64, device=dev)
    status = torch.zeros((), dtype=torch.int32, device=dev)
    for e in range(E):
        experts[e].see(priors[e])

    def step():
        with torch.no_grad():
            gating_probs = torch.exp(gating(image))                                          # test_esac.py:163
            e_hyps = torch.multinomial(gating_probs[0], M, replacement=True)                 # :173 (no .cpu())
            prediction = torch.stack([experts[e](image)[0] for e in range(E)])               # :179-185
        esac_api.forward_async(prediction, e_hyps, shift, camera, opt.threshold, opt.inlieralpha, opt.inlierbeta,
                               opt.maxreprojection, OUTPUT_SUBSAMPLE, pose, expert, status)  # :192-205
        return prediction, e_hyps

    esac_api.reserve_forward_async(1, E, H, W, M, OUTPUT_SUBSAMPLE)
    side = torch.cuda.Stream()            # warm up torch's kernels off the default stream, as torch.cuda.graph expects
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        prediction, e_hyps = step()
    esac_api.set_seed(2020)   # resets the eager and the stream-ordered call counters alike

    failures = 0
    rot_errs, trans_errs = [], []
    t_total = 0.0
    for i in range(len(testset)):
        idx, img, focallength, gt_pose, _, _ = testset[i]
        image.copy_(img[None])
        priors.copy_(testset.prediction_for(int(idx)))
        camera.copy_(torch.tensor([float(focallength), img.size(2) / 2, img.size(1) / 2]))   # :147-150
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.replay()
        out = pose.cpu().numpy()
        t_total += time.perf_counter() - t0
        if int(status) != 0:
            print(f"image {i}: bad expert index in the assignment")
            failures += 1
            continue
        rot, trans = pose_error(out, gt_pose.numpy())                                         # :209-222
        rot_errs.append(rot)
        trans_errs.append(trans)
        line = f"image {i}: f = {float(focallength):7.1f}, expert {int(expert)}, rot {rot:.3f} deg, trans {100 * trans:.2f} cm"
        if opt.check:
            # eager call i on the graph's own coordinates and assignment draws what replay i drew
            ref = torch.zeros(4, 4, device=dev)
            ref_e = esac.forward(prediction, e_hyps, ref, 0, 0, float(focallength), img.size(2) / 2, img.size(1) / 2,
                                 opt.threshold, opt.inlieralpha, opt.inlierbeta, opt.maxreprojection, OUTPUT_SUBSAMPLE)
            same = ref_e == int(expert) and np.array_equal(ref.cpu().numpy(), out)
            line += ", eager: " + ("bitwise equal" if same else "DIFFERENT")
            failures += not same
        print(line, flush=True)
    if rot_errs:
        print(f"median rot {np.median(rot_errs):.3f} deg, median trans {100 * np.median(trans_errs):.2f} cm, "
              f"{1e3 * t_total / len(testset):.2f} ms per image (replay + pose read-back)")
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
