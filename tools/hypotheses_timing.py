"""Times one training step's loss and coordinate gradient two ways, on CUDA tensors (GPU only):
  esac_loss                       esac.backward as one autograd node (the reference loss inside the library);
  esac_hypotheses + torch loss    the hypotheses node, reference_pose_loss, softmax and the expectation in torch, backward().
Both compute the same loss and gradient.  Shapes: the bench workload (E = 7, M = 256, 480x640 cells) and 60x80 cells with
E = 20, M = 1024.  Prints the card name and power limit first, then the median of --reps timed steps per variant.

    python tools/hypotheses_timing.py --reps 20
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
from esac_b200.autograd import esac_hypotheses, esac_loss, reference_pose_loss  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

SHAPES = [("bench 480x640 E=7 M=256", dict(E=7, H=480, W=640, M=256, sub=1, seed=2)),
          ("60x80 E=20 M=1024", dict(E=20, H=60, W=80, M=1024, sub=8, seed=1))]
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
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print(f"card: {card()}", flush=True)
    api.context().set_option("fixed_seed", 1)
    for name, kw in SHAPES:
        sc = make_scene(**kw)
        coords0 = torch.from_numpy(sc.coords).cuda()
        assign = torch.from_numpy(sc.assign).cuda()
        gt = torch.from_numpy(sc.gt_pose).cuda()
        gating = torch.zeros(1, sc.coords.shape[0], device="cuda", requires_grad=True)

        def library_loss():
            coords = coords0.clone().requires_grad_(True)
            api.set_seed(5)
            esac_loss(coords, gating, assign, gt, *W_LOSS, *sc.params).backward()
            return coords.grad

        def torch_loss():
            coords = coords0.clone().requires_grad_(True)
            api.set_seed(5)
            scores, poses, _ = esac_hypotheses(coords, assign, *sc.params)
            (torch.softmax(scores, 0) * reference_pose_loss(poses, gt, *W_LOSS)).sum().backward()
            return coords.grad

        g1, g2 = library_loss(), torch_loss()
        rel = float((g1 - g2).abs().max() / g1.abs().max())
        t1, t2 = timed(library_loss, args.reps, args.warmup), timed(torch_loss, args.reps, args.warmup)
        print(json.dumps({"shape": name, "esac_loss_ms": round(t1[0], 3), "esac_loss_ms_range": [round(t1[1], 3), round(t1[2], 3)],
                          "hypotheses_plus_torch_loss_ms": round(t2[0], 3),
                          "hypotheses_plus_torch_loss_ms_range": [round(t2[1], 3), round(t2[2], 3)],
                          "grad_rel_diff": rel, "n_contrib": api.last_stats()["n_contrib"]}), flush=True)


if __name__ == "__main__":
    main()
