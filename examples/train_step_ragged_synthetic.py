"""A batched train_esac.py step (code/train_esac.py:105-183) over a batch of images of different sizes, each with its own
camera, as on 19Scenes, Aachen or Dubrovnik, where every image keeps its own aspect ratio (datasets/setup_aachen.py resizes
to a 480-pixel short side).

The batch mixes landscape and portrait maps (60x80, 80x60, 60x90, 61x107 cells).  Stand-in networks: each expert is a
learnable per-channel affine map of the scene-coordinate prior that esac_b200.synth.make_scene generates, and the gating head
is a linear layer on fixed features.  The whole batch goes through one `esac_loss_batch` call on a list of maps; with
--check every step is compared with a loop of single-image `esac_loss` calls on a copy of the networks: the losses, the
gradient of every map and the parameters after the Adam step must agree exactly.

    python examples/train_step_ragged_synthetic.py --steps 3 --check
"""
from __future__ import annotations

import argparse
import copy
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import esac_loss, esac_loss_batch  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

SHAPES = [(60, 80), (80, 60), (60, 90), (61, 107)]
FOCAL = [525.0, 610.5, 480.25, 733.0]


class Nets(nn.Module):
    def __init__(self, E, feats):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(E, 3, 1, 1))
        self.shift = nn.Parameter(torch.zeros(E, 3, 1, 1))
        self.gating = nn.Linear(feats, E)

    def forward(self, priors, feats):
        return [p * self.scale + self.shift for p in priors], torch.log_softmax(self.gating(feats), 1)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--hypotheses", type=int, default=64)
    ap.add_argument("--check", action="store_true", help="compare every step with a loop of single-image esac_loss calls")
    args = ap.parse_args()
    E, M, B = args.experts, args.hypotheses, len(SHAPES)
    torch.manual_seed(0)
    nets = Nets(E, 16).cuda()
    twin = copy.deepcopy(nets) if args.check else None
    opt = torch.optim.Adam(nets.parameters(), lr=1e-3)
    opt_twin = torch.optim.Adam(twin.parameters(), lr=1e-3) if args.check else None
    api.context().set_option("fixed_seed", 0)
    for step in range(args.steps):
        scenes = [make_scene(E=E, H=h, W=w, M=M, sub=8, seed=1000 * step + b, f=FOCAL[b], shiftX=(b * 3) % 7 - 3,
                             shiftY=(b * 5) % 7 - 3) for b, (h, w) in enumerate(SHAPES)]
        gen = torch.Generator().manual_seed(step)
        priors = [torch.from_numpy(s.coords).cuda() + 0.01 * torch.randn(s.coords.shape, generator=gen).cuda() for s in scenes]
        feats = torch.randn(B, 16, generator=gen).cuda()
        assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
        gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
        cams = tuple([getattr(s, k) for s in scenes] for k in ("shiftX", "shiftY", "f", "ppx", "ppy"))
        params = (1.0, 100.0, 100.0) + cams + scenes[0].params[5:]
        seed = 7 + step
        t0 = time.perf_counter()
        opt.zero_grad()
        preds, lp = nets(priors, feats)
        for p in preds:
            p.retain_grad()
        api.set_seed(seed)
        losses = esac_loss_batch(preds, lp, assign, gts, *params)
        losses.sum().backward()
        grads = [p.grad.clone() for p in preds]
        opt.step()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        line = f"step {step}: losses {[round(v, 4) for v in losses.tolist()]}, {ms:.1f} ms"
        if args.check:
            opt_twin.zero_grad()
            preds1, lp1 = twin(priors, feats)
            for p in preds1:
                p.retain_grad()
            api.set_seed(seed)
            ref = [esac_loss(preds1[b], lp1[b], assign[b], gts[b], 1.0, 100.0, 100.0, *scenes[b].params) for b in range(B)]
            sum(ref).backward()
            opt_twin.step()
            assert losses.tolist() == [r.item() for r in ref], (losses.tolist(), [r.item() for r in ref])
            for b in range(B):
                assert torch.equal(grads[b], preds1[b].grad), f"step {step}: gradient of image {b} differs"
            for a, c in zip(nets.parameters(), twin.parameters()):
                assert torch.equal(a, c), f"step {step}: parameters differ after the Adam step"
            line += ", matches the per-image loop"
        print(line)
    if args.check:
        print("check ok")
    return 0


if __name__ == "__main__":
    sys.exit(main())
