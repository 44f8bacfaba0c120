"""Times one training step (loss + backward()) of a batch on CUDA tensors three ways (GPU only):
  (a) loop      esac_hypotheses per image, softmax . reference_pose_loss in torch;
  (b) batch     esac_hypotheses_batch on the whole batch, the same torch loss;
  (c) library   esac_loss_batch (the reference loss inside the library, api.backward_batch's worker streams).
All three compute the same losses and gradients; the tool prints whether (a) and (b) give bitwise the same gradients and the
largest relative gradient difference of (b) against (c).  Workloads: 8 images at 60x80 cells (the reference's training
resolution, expert.py:13) with E = 7, M = 256; the Aachen-like ragged batch of tools/ragged_batch_timing.py (8 maps in 5
shapes, E = 10, M = 256); 4 images at 480x640 cells, E = 7, M = 256.  Prints the card name and power limit first, then the
median, minimum and maximum over --reps timed steps per variant.

    python tools/hypotheses_batch_timing.py --reps 20
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import esac_hypotheses, esac_hypotheses_batch, esac_loss_batch, reference_pose_loss  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

AACHEN = [(60, 80), (80, 60), (60, 90), (60, 80), (90, 60), (60, 107), (60, 80), (80, 60)]
WORKLOADS = [("8 x 60x80 E=7 M=256", [(60, 80)] * 8, dict(E=7, M=256, sub=8)),
             ("Aachen-like ragged 8 maps E=10 M=256", AACHEN, dict(E=10, M=256, sub=8)),
             ("4 x 480x640 E=7 M=256", [(480, 640)] * 4, dict(E=7, M=256, sub=1))]
W_LOSS = (1.0, 100.0, 100.0)


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = ""
    return q or torch.cuda.get_device_name()


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return [round(float(np.median(ms)), 3), round(float(np.min(ms)), 3), round(float(np.max(ms)), 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print(f"card: {card()}", flush=True)
    api.context().set_option("fixed_seed", 0)
    for name, shapes, kw in WORKLOADS:
        scenes = [make_scene(H=h, W=w, seed=b, f=500.0 + 10 * b, shiftX=b % 3, shiftY=(2 * b) % 5, **kw)
                  for b, (h, w) in enumerate(shapes)]
        B = len(scenes)
        coords0 = [torch.from_numpy(s.coords).cuda() for s in scenes]
        assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
        gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
        params = [[getattr(s, k) for s in scenes] for k in ("shiftX", "shiftY", "f", "ppx", "ppy")] + list(scenes[0].params[5:])
        gating = torch.zeros(B, kw["E"], device="cuda", requires_grad=True)

        def loop():
            coords = [c.clone().requires_grad_(True) for c in coords0]
            api.set_seed(5)
            total = 0
            for b in range(B):
                scores, poses, _ = esac_hypotheses(coords[b], assign[b], *scenes[b].params)
                total = total + (torch.softmax(scores, 0) * reference_pose_loss(poses, gts[b], *W_LOSS)).sum()
            total.backward()
            return [c.grad for c in coords]

        def batch():
            coords = [c.clone().requires_grad_(True) for c in coords0]
            api.set_seed(5)
            scores, poses, _ = esac_hypotheses_batch(coords, assign, *params)
            (torch.softmax(scores, 1) * reference_pose_loss(poses, gts, *W_LOSS)).sum().backward()
            return [c.grad for c in coords]

        def library():
            coords = [c.clone().requires_grad_(True) for c in coords0]
            api.set_seed(5)
            esac_loss_batch(coords, gating, assign, gts, *W_LOSS, *params).sum().backward()
            return [c.grad for c in coords]

        ga, gb, gc = loop(), batch(), library()
        bitwise = all(torch.equal(x, y) for x, y in zip(ga, gb))
        rel = max(float((x - y).abs().max() / y.abs().max()) for x, y in zip(gb, gc))
        res = {"workload": name, "B": B}
        for label, fn in (("loop", loop), ("batch", batch), ("esac_loss_batch", library)):
            res[label + "_ms"] = timed(fn, args.reps, args.warmup)  # [median, min, max]
        res.update({"loop_vs_batch_grads_bitwise": bitwise, "batch_vs_esac_loss_batch_grad_rel_diff": rel})
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
