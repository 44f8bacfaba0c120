"""custom_loss_step_synthetic.py on a batch: one DSAC*-loss training step over B images of different sizes, each with its
own camera and shift, through the batched hypotheses node.

`esac_hypotheses_batch` takes the list of the experts' maps and returns the soft-inlier scores [B,M] and refined poses
[B,M,6] of the hypotheses esac_loss_batch would draw; the images run on the library's worker streams, so their host
synchronisations overlap.  The loss is DSAC*'s per-hypothesis `max(angle in degrees, translation error in cm)`, its
expectation over each image's softmax is left to autograd, and the batch loss is the sum over the images.  Hypotheses
are assigned with `api.assign_hypotheses`, whose histogram gives the trainer's REINFORCE term per image: the gradient of
image b's gating log-probabilities is `loss_b * histogram(e_hyps[b])`.

Stand-in networks as in custom_loss_step_synthetic.py.  With --check every step also runs the reference loss through the
batched node, `softmax(scores, 1) . reference_pose_loss(poses, gts, ...)`, and compares each image's loss and coordinate
gradient with `esac_loss_batch` on the same hypotheses.

    python examples/custom_loss_batch_step_synthetic.py --steps 3 --check
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import esac_hypotheses_batch, esac_loss_batch, pose_to_transform, reference_pose_loss  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

REF_LOSS = (1.0, 100.0, 100.0)  # wLossRot, wLossTrans, lossCut of the reference trainer
SHAPES = [(60, 80), (80, 60), (60, 90), (90, 60)]  # 480-pixel short side at sub-sampling 8, landscape and portrait


class Nets(nn.Module):
    def __init__(self, E, feats):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(E, 3, 1, 1))
        self.shift = nn.Parameter(torch.zeros(E, 3, 1, 1))
        self.gating = nn.Linear(feats, E)

    def forward(self, priors, feats):
        return [p * self.scale + self.shift for p in priors], torch.log_softmax(self.gating(feats), 1)


def dsac_star_loss(T, gt):
    """max(rotation error in degrees, translation error in cm) of camera->world transforms T [B,M,4,4] against gt [B,4,4]."""
    cos = ((T[..., :3, :3] * gt[:, None, :3, :3]).sum((-2, -1)) - 1) / 2
    angle = torch.rad2deg(torch.acos(cos.clamp(-1 + 1e-12, 1 - 1e-12)))
    trans_cm = 100 * (T[..., :3, 3] - gt[:, None, :3, 3]).norm(dim=-1)
    return torch.maximum(angle, trans_cm)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--hypotheses", type=int, default=64)
    ap.add_argument("--check", action="store_true", help="compare the reference loss through the node with esac_loss_batch")
    args = ap.parse_args()
    E, M, B = args.experts, args.hypotheses, len(SHAPES)
    torch.manual_seed(0)
    nets = Nets(E, 16).cuda()
    opt = torch.optim.Adam(nets.parameters(), lr=1e-3)
    api.context().set_option("fixed_seed", 0)
    for step in range(args.steps):
        rng = np.random.default_rng(step)
        shifts = rng.integers(0, 8, size=(B, 2))  # train_esac.py:125: a random shift per image
        scenes = [make_scene(E=E, H=h, W=w, M=M, sub=8, seed=3000 + 10 * step + b, outlier_frac=0.6, f=500.0 + 10 * b,
                             ppx=4 * w + b, ppy=4 * h - b, shiftX=int(shifts[b, 0]), shiftY=int(shifts[b, 1]))
                  for b, (h, w) in enumerate(SHAPES)]
        gen = torch.Generator().manual_seed(step)
        priors = [torch.from_numpy(s.coords).cuda() + 0.01 * torch.randn(s.coords.shape, generator=gen).cuda() for s in scenes]
        feats = torch.randn(B, 16, generator=gen).cuda()
        gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
        params = [[getattr(s, k) for s in scenes] for k in ("shiftX", "shiftY", "f", "ppx", "ppy")] + list(scenes[0].params[5:])
        seed = 11 + step
        t0 = time.perf_counter()
        opt.zero_grad()
        prediction, log_probs = nets(priors, feats)
        e_hyps, hist = api.assign_hypotheses(torch.exp(log_probs.detach()), M, seed=100 + step)    # train_esac.py:130-141
        api.set_seed(seed)
        scores, poses, contributing = esac_hypotheses_batch(prediction, e_hyps, *params)
        losses = (torch.softmax(scores, 1) * dsac_star_loss(pose_to_transform(poses), gts.double())).sum(1)
        # the gating gradient of the trainer per image (train_esac.py:171-176): d/d log_probs[b] = loss_b * histogram(e_hyps[b])
        total = losses.sum() + (losses.detach()[:, None] * hist * log_probs).sum()
        total.backward()
        opt.step()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        line = (f"step {step}: expected DSAC* losses {[round(v, 3) for v in losses.tolist()]}, "
                f"{contributing.sum(1).tolist()} contributing hypotheses, {ms:.1f} ms")
        if args.check:
            coords = [p.detach().clone().requires_grad_(True) for p in prediction]
            api.set_seed(seed)
            sc_, po_, _ = esac_hypotheses_batch(coords, e_hyps, *params)
            mine = (torch.softmax(sc_, 1) * reference_pose_loss(po_, gts, *REF_LOSS)).sum(1)
            mine.sum().backward()
            ref_coords = [p.detach().clone().requires_grad_(True) for p in prediction]
            gating = log_probs.detach().clone().requires_grad_(True)
            api.set_seed(seed)
            ref = esac_loss_batch(ref_coords, gating, e_hyps, gts, *REF_LOSS, *params)
            ref.sum().backward()
            # the float64 values behind esac_loss_batch's float32 output: the same call once more
            api.set_seed(seed)
            ref_losses = api.backward_batch([p.detach() for p in prediction], [torch.zeros_like(p) for p in prediction], e_hyps,
                                            gts, *REF_LOSS, *params)
            assert torch.equal(ref.detach(), ref.new_tensor(ref_losses))
            worst_l = worst_g = 0.0
            for b in range(B):
                dl = abs(mine[b].item() - ref_losses[b])
                dg = (coords[b].grad - ref_coords[b].grad).abs().max().item()
                scale = ref_coords[b].grad.abs().max().item()
                assert dl <= 1e-12 * abs(ref_losses[b]), f"step {step} image {b}: loss {mine[b].item()} against {ref_losses[b]}"
                assert scale > 0 and dg <= 1e-6 * scale, f"step {step} image {b}: gradient differs by {dg} (largest {scale})"
                worst_l, worst_g = max(worst_l, dl / abs(ref_losses[b])), max(worst_g, dg / scale)
            line += (f", reference loss through the node matches esac_loss_batch (largest relative loss diff {worst_l:.1e}, "
                     f"grad diff {worst_g:.1e})")
        print(line)
    if args.check:
        print("check ok")
    return 0


if __name__ == "__main__":
    sys.exit(main())
