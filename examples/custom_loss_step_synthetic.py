"""A train_esac.py step (code/train_esac.py:105-183) with a pose loss written in torch instead of the reference's.

The hypotheses come from `esac_hypotheses`, a differentiable function of the scene coordinates: soft-inlier scores and refined
poses of the hypotheses esac.backward would draw.  The loss is DSAC*'s per-hypothesis `max(angle in degrees, translation
error in cm)` on `pose_to_transform(poses)`, and the expectation over the softmax of the scores is left to autograd.  The
gating network gets the trainer's REINFORCE term: the gradient of its log-probabilities is `loss * histogram(e_hyps)`.

Stand-in networks as in train_step_ragged_synthetic.py: each expert is a learnable per-channel affine map of the
scene-coordinate prior from esac_b200.synth.make_scene, and the gating head is a linear layer on fixed features.  With --check
every step also runs the reference loss through the same node, `softmax(scores) . reference_pose_loss(poses, ...)`, and
compares loss and coordinate gradient with `esac_loss` (esac.backward) on the same hypotheses.

    python examples/custom_loss_step_synthetic.py --steps 3 --check
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import torch
import torch.nn as nn

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import esac_hypotheses, esac_loss, pose_to_transform, reference_pose_loss  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

REF_LOSS = (1.0, 100.0, 100.0)  # wLossRot, wLossTrans, lossCut of the reference trainer


class Nets(nn.Module):
    def __init__(self, E, feats):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(E, 3, 1, 1))
        self.shift = nn.Parameter(torch.zeros(E, 3, 1, 1))
        self.gating = nn.Linear(feats, E)

    def forward(self, prior, feats):
        return prior * self.scale + self.shift, torch.log_softmax(self.gating(feats), 1)


def dsac_star_loss(T, gt):
    """max(rotation error in degrees, translation error in cm) of camera->world transforms T [M,4,4] against gt [4,4]."""
    cos = ((T[:, :3, :3] * gt[:3, :3]).sum((1, 2)) - 1) / 2
    angle = torch.rad2deg(torch.acos(cos.clamp(-1 + 1e-12, 1 - 1e-12)))
    trans_cm = 100 * (T[:, :3, 3] - gt[:3, 3]).norm(dim=1)
    return torch.maximum(angle, trans_cm)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--experts", type=int, default=4)
    ap.add_argument("--hypotheses", type=int, default=64)
    ap.add_argument("--check", action="store_true", help="compare the reference loss through the node with esac_loss")
    args = ap.parse_args()
    E, M = args.experts, args.hypotheses
    torch.manual_seed(0)
    nets = Nets(E, 16).cuda()
    opt = torch.optim.Adam(nets.parameters(), lr=1e-3)
    api.context().set_option("fixed_seed", 0)
    for step in range(args.steps):
        sc = make_scene(E=E, H=60, W=80, M=M, sub=8, seed=2000 + step, outlier_frac=0.6)
        gen = torch.Generator().manual_seed(step)
        prior = torch.from_numpy(sc.coords).cuda() + 0.01 * torch.randn(sc.coords.shape, generator=gen).cuda()
        feats = torch.randn(1, 16, generator=gen).cuda()
        gt = torch.from_numpy(sc.gt_pose).cuda()
        seed = 11 + step
        t0 = time.perf_counter()
        opt.zero_grad()
        prediction, log_probs = nets(prior, feats)
        e_hyps = torch.multinomial(torch.exp(log_probs.detach()[0]).cpu(), M, replacement=True)      # train_esac.py:138
        hist = torch.histc(e_hyps.float(), bins=E, min=0, max=E - 1).cuda()                        # :141
        api.set_seed(seed)
        scores, poses, contributing = esac_hypotheses(prediction, e_hyps.cuda(), *sc.params)
        loss = (torch.softmax(scores, 0) * dsac_star_loss(pose_to_transform(poses), gt.double())).sum()
        # the gating gradient of the trainer (train_esac.py:171-176): d/d log_probs = loss * histogram(e_hyps)
        total = loss + (loss.detach() * hist * log_probs[0]).sum()
        total.backward()
        opt.step()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        line = (f"step {step}: expected DSAC* loss {loss.item():.3f}, {int(contributing.sum())} contributing hypotheses, "
                f"{ms:.1f} ms")
        if args.check:
            coords = prediction.detach().clone().requires_grad_(True)
            api.set_seed(seed)
            sc_, po_, _ = esac_hypotheses(coords, e_hyps.cuda(), *sc.params)
            mine = (torch.softmax(sc_, 0) * reference_pose_loss(po_, gt, *REF_LOSS)).sum()
            mine.backward()
            ref_coords = prediction.detach().clone().requires_grad_(True)
            gating = log_probs.detach().clone().requires_grad_(True)
            api.set_seed(seed)
            ref = esac_loss(ref_coords, gating, e_hyps.cuda(), gt, *REF_LOSS, *sc.params)
            ref_loss = api.last_stats()["expected_loss"]  # the float64 value behind esac_loss's float32 output
            ref.backward()
            dl = abs(mine.item() - ref_loss)
            dg = (coords.grad - ref_coords.grad).abs().max().item()
            scale = ref_coords.grad.abs().max().item()
            assert dl <= 1e-12 * abs(ref_loss), f"step {step}: loss {mine.item()} against esac_loss {ref_loss}"
            assert scale > 0 and dg <= 1e-6 * scale, f"step {step}: gradient differs by {dg} (largest entry {scale})"
            line += f", reference loss through the node matches esac_loss (loss diff {dl:.1e}, grad diff {dg / scale:.1e})"
        print(line)
    if args.check:
        print("check ok")
    return 0


if __name__ == "__main__":
    sys.exit(main())
