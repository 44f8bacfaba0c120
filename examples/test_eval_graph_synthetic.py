"""The reference's whole test loop (code/test_esac.py:137-293) with its evaluation on the device: the gated test step of
examples/test_step_gated_graph_synthetic.py, captured once, with esac_b200.evaluate.PoseEvaluator.update inside the graph.

Every replay appends the image's record (pose errors, correct expert, experts active, pose-file entry) to the evaluator's
store on the device, so the loop never waits for the GPU: the inputs of every image sit in pinned host memory and reach
the graph's static inputs through non_blocking copies, and the host reads nothing until the last image is enqueued.  Then
one read-back gives the reference's table, results file and pose file.

    python examples/test_eval_graph_synthetic.py --images 16 --experts 6 --outdir /tmp/esac_eval --check

--check keeps a device copy of every replay's pose, expert and status (stream-ordered, no synchronisation), reads them
back at the end, evaluates them on the host with the float64 restatement in oracle/eval_oracle.py and compares the
records, the table and the pose-file lines.
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
import esac_b200.api as esac_api  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE  # noqa: E402
from esac_b200.evaluate import PoseEvaluator  # noqa: E402
from esac_b200.gate import ExpertGate  # noqa: E402
from test_step_graph_synthetic import PerImageFocalDataset  # noqa: E402
from train_step_synthetic import TinyExpert, TinyGating  # noqa: E402

SEED0 = 4242   # the draw's seed at the first replay; every replay adds 1


def options(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--distinct", type=int, default=0, help="cycle through this many generated images (0: all distinct)")
    ap.add_argument("--experts", type=int, default=6)
    ap.add_argument("--hypotheses", "-hyps", type=int, default=256)     # test_esac.py:29
    ap.add_argument("--maxexperts", type=int, default=2, help="util.clamp_probs: draw from the n most likely experts (-1: all)")
    ap.add_argument("--threshold", type=float, default=10)              # :32
    ap.add_argument("--inlieralpha", type=float, default=100)           # :35
    ap.add_argument("--inlierbeta", type=float, default=0.5)            # :38
    ap.add_argument("--maxreprojection", type=float, default=100)       # :41
    ap.add_argument("--rotthreshold", type=float, default=5)            # :56
    ap.add_argument("--transthreshold", type=float, default=5)          # :59
    ap.add_argument("--outdir", type=str, default=None, help="write results_esac_synthetic.txt and poses_esac_synthetic.txt here")
    ap.add_argument("--check", action="store_true", help="compare with host evaluation of the read-back poses")
    return ap.parse_args(argv)


class GatedTestStep:
    """The captured test step: gating, hypothesis draw, the experts with hypotheses, forward_async, and (evaluate=True) the
    evaluator's update.  Its static inputs are filled from pinned host memory by load(i)."""

    def __init__(self, opt, evaluate: bool = True):
        torch.backends.cudnn.deterministic = True
        torch.backends.cudnn.benchmark = False
        dev = torch.device("cuda")
        E, M = opt.experts, opt.hypotheses
        n_gen = opt.distinct if 0 < opt.distinct < opt.images else opt.images
        testset = PerImageFocalDataset(num_experts=E, length=n_gen, hypotheses=M, seed=11, training=False)
        H, W = testset.image_hw[0] // OUTPUT_SUBSAMPLE, testset.image_hw[1] // OUTPUT_SUBSAMPLE
        torch.manual_seed(0)
        experts = [TinyExpert().to(dev).eval() for _ in range(E)]
        gating = TinyGating(E).to(dev).eval()
        thresholds = (opt.threshold, opt.inlieralpha, opt.inlierbeta, opt.maxreprojection, OUTPUT_SUBSAMPLE)
        self.n_gen = n_gen
        self.names = [f"synthetic/frame-{i:06d}" for i in range(opt.images)]   # util.strip_file_name's form

        # every generated image's inputs in pinned host memory: nothing is written there while copies are in flight
        self.h_image = torch.empty(n_gen, 1, 1, *testset.image_hw).pin_memory()
        self.h_priors = torch.empty(n_gen, E, 3, H, W).pin_memory()
        self.h_camera = torch.empty(n_gen, 3).pin_memory()
        self.h_gt = torch.empty(n_gen, 4, 4).pin_memory()
        self.h_scene = torch.empty(n_gen, dtype=torch.int64).pin_memory()
        for i in range(n_gen):
            idx, img, focallength, gt_pose, _, gt_expert = testset[i]
            self.h_image[i, 0].copy_(img)
            self.h_priors[i].copy_(testset.prediction_for(int(idx)))
            self.h_camera[i] = torch.tensor([float(focallength), img.size(2) / 2, img.size(1) / 2])   # :145-147
            self.h_gt[i].copy_(gt_pose)
            self.h_scene[i] = int(gt_expert)

        # static inputs and outputs of the graph
        self.image = torch.zeros(1, 1, *testset.image_hw, device=dev)
        self.priors = torch.zeros(E, 3, H, W, device=dev)
        self.camera = torch.zeros(3, device=dev)
        self.gt_pose = torch.zeros(4, 4, device=dev)
        self.gt_scene = torch.zeros((), dtype=torch.int64, device=dev)
        shift = torch.zeros(2, dtype=torch.int32, device=dev)
        self.seed = torch.tensor([SEED0], dtype=torch.int64, device=dev)
        e_hyps = torch.zeros(M, dtype=torch.int64, device=dev)
        self.hist = torch.zeros(E, device=dev)
        draw_status = torch.zeros((), dtype=torch.int32, device=dev)
        prediction = torch.zeros(E, 3, H, W, device=dev)
        self.pose = torch.zeros(4, 4, device=dev)
        self.expert = torch.zeros((), dtype=torch.int64, device=dev)
        self.status = torch.zeros((), dtype=torch.int32, device=dev)
        for e in range(E):
            experts[e].see(self.priors[e])
        gate = ExpertGate(E)
        self.evaluator = PoseEvaluator(E, opt.images) if evaluate else None

        def step():
            with torch.no_grad():
                gating_probs = torch.exp(gating(self.image))[0]                                         # :163
                esac_api.assign_hypotheses_async(gating_probs, M, self.seed, e_hyps, self.hist, draw_status,
                                                 maxExperts=opt.maxexperts)                             # :165-178
                self.seed.add_(1)
                gate.arm(self.hist)
                prediction.zero_()
                for e in range(E):                                                                      # :183-185
                    gate.run(e, lambda e=e: prediction[e].copy_(experts[e](self.image)[0]))
            esac_api.forward_async(prediction, e_hyps, shift, self.camera, *thresholds, self.pose, self.expert,
                                   self.status)                                                         # :192-205
            if self.evaluator is not None:                                                              # :209-247
                self.evaluator.update(self.pose, self.gt_pose, self.expert, self.gt_scene, hist=self.hist,
                                      status=self.status)

        # the graph reads and writes these tensors and modules at every replay: they must live as long as it does
        self.keep = (experts, gating, gate, shift, e_hyps, draw_status, prediction, step)
        esac_api.reserve_forward_async(1, E, H, W, M, OUTPUT_SUBSAMPLE)
        self.load(0)
        side = torch.cuda.Stream()            # warm up torch's kernels off the default stream, as torch.cuda.graph expects
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step()
        torch.cuda.current_stream().wait_stream(side)
        self.graph = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(self.graph):
            step()
        gate.finalize(self.graph)
        self.reset()

    def reset(self):
        """Back to the first replay's seed and an empty store, stream-ordered."""
        self.seed.fill_(SEED0)
        if self.evaluator is not None:
            self.evaluator.reset()
        esac_api.set_seed(2020)

    def load(self, i: int):
        """Image i's inputs into the graph's static inputs: non_blocking copies from pinned memory."""
        j = i % self.n_gen
        self.image.copy_(self.h_image[j], non_blocking=True)
        self.priors.copy_(self.h_priors[j], non_blocking=True)
        self.camera.copy_(self.h_camera[j], non_blocking=True)
        self.gt_pose.copy_(self.h_gt[j], non_blocking=True)
        self.gt_scene.copy_(self.h_scene[j], non_blocking=True)

    def gt(self, i: int):
        j = i % self.n_gen
        return self.h_gt[j].numpy(), int(self.h_scene[j])


def run(opt) -> dict:
    """The loop; returns the evaluator's records, table and pose lines, and with opt.check the host evaluation's."""
    t = GatedTestStep(opt)
    dev = t.pose.device
    if opt.check:
        kept = torch.zeros(opt.images, 4, 4, device=dev), torch.zeros(opt.images, dtype=torch.int64, device=dev), \
            torch.zeros(opt.images, dtype=torch.int32, device=dev), torch.zeros(opt.images, opt.experts, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(opt.images):
        t.load(i)
        t.graph.replay()
        if opt.check:
            for dst, src in zip(kept, (t.pose, t.expert, t.status, t.hist)):
                dst[i].copy_(src)
    records = t.evaluator.records()                    # the one read-back
    seconds = time.perf_counter() - t0
    out = {"records": records, "names": t.names, "seconds": seconds,
           "table": t.evaluator.table(opt.rotthreshold, opt.transthreshold, average=True),
           "pose_lines": t.evaluator.pose_lines(t.names)}
    if opt.check:
        from oracle import eval_oracle as O
        poses, experts, status, hist = (k.cpu().numpy() for k in kept)
        gts = [t.gt(i) for i in range(opt.images)]
        host = O.evaluate_batch(poses, np.stack([g for g, _ in gts]), experts, [s for _, s in gts], hist, status)
        out["host_records"] = host
        out["host_table"] = O.table(host, opt.experts, opt.rotthreshold, opt.transthreshold, average=True)
        out["host_pose_lines"] = [O.pose_line(n, r) for n, r in zip(t.names, host)]
    return out


def main(argv=None):
    opt = options(argv)
    r = run(opt)
    t = r["table"]
    print("\n".join(t["console"]))
    print("\n" + t["experts"][0])
    print(t["experts"][1])
    if t["excluded"]:
        print(f"{t['excluded']} image(s) left out: forward status != 0 or scene outside [0, {opt.experts})")
    print(f"\n{1e3 * r['seconds'] / opt.images:.3f} ms per image (pinned inputs, replay with evaluation, one read-back)")
    if opt.outdir:
        d = Path(opt.outdir)
        d.mkdir(parents=True, exist_ok=True)
        (d / "results_esac_synthetic.txt").write_text("".join(line + "\n" for line in t["results"]))
        (d / "poses_esac_synthetic.txt").write_text("".join(line + "\n" for line in r["pose_lines"]))
    if opt.check:
        h = r["host_table"]
        same = (t["console"], t["results"], t["experts"], t["excluded"]) == (h["console"], h["results"], h["experts"],
                                                                             h["excluded"])
        same = same and r["pose_lines"] == r["host_pose_lines"]
        print("host evaluation of the read-back poses: " + ("same table and pose file" if same else "DIFFERENT"))
        return 0 if same else 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
