"""HBM roofline of the fused scene-coordinate loss (esac_b200/csrc/coord_loss.cu).

Algorithmic bytes per cell with the gradient: 48 B = count pass 12 B (ground truth read) + loss pass 24 B read (prediction
and ground truth) + 12 B written (gradient); loss only: 24 B.  Prints the kernel time (CUDA events around the kernels, the
library's own stage timer `ms_score`), the algorithmic GB/s and its share of the H100 SXM data-sheet peak of 3.35 TB/s, the
wall time of the whole call (one host synchronisation included), and beside them the torch op sequence of
init_expert.py:114-132 plus autograd on one image.  Needs a GPU; prints the card name and power limit first."""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import esac_b200.api as api  # noqa: E402

PEAK_GBS = 3350.0   # H100 SXM data sheet, HBM3


def torch_ref(pred, gt, cut):
    """The original op sequence on CUDA tensors (batch of 1, as the reference trains)."""
    p = pred.detach().clone().requires_grad_(True)
    prediction = p.squeeze().contiguous().view(3, -1)
    gt_coords = gt.squeeze().contiguous().view(3, -1)
    coords_mask = gt_coords.abs().sum(0) != 0
    prediction = prediction[:, coords_mask]
    gt_coords = gt_coords[:, coords_mask]
    loss = torch.norm(prediction - gt_coords, dim=0)
    loss_l1 = loss[loss <= cut]
    loss_sqrt = torch.sqrt(cut * loss[loss > cut])
    robust_loss = (loss_l1.sum() + loss_sqrt.sum()) / float(loss.size(0))
    robust_loss.backward()
    return robust_loss, p.grad


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    if not torch.cuda.is_available():
        raise SystemExit("coord_loss_bandwidth: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {q.stdout.strip() or torch.cuda.get_device_name()}")
    ctx = api.context()
    cut = 100.0
    g = torch.Generator(device="cuda").manual_seed(5)
    for (H, W) in [(60, 80), (480, 640)]:
        for B in (1, 8, 64):
            gt = torch.randn((B, 3, H, W), device="cuda", generator=g) * 2.0
            gt *= (torch.rand((B, 1, H, W), device="cuda", generator=g) < 0.7)       # 30 % cells without ground truth
            pred = gt + 50.0 * torch.randn((B, 3, H, W), device="cuda", generator=g)
            grads = torch.empty_like(pred)
            cells = B * H * W
            line = f"B={B:3d} {H}x{W}:"
            for with_grad, nbytes in ((True, 48), (False, 24)):
                ms, wall = [], []
                for it in range(40):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    api.coord_loss(pred, gt, cut, outGradients=grads if with_grad else None)
                    wall.append((time.perf_counter() - t0) * 1e3)
                    ms.append(ctx.stats()["ms_score"])
                k, wl = median(ms[5:]), median(wall[5:])
                gbs = cells * nbytes / k / 1e6
                line += (f"  {'loss+grad' if with_grad else 'loss only'} ({nbytes} B/cell): kernels {k * 1e3:7.1f} us "
                         f"{gbs:7.1f} GB/s ({gbs / PEAK_GBS:.2f} of peak), call wall {wl * 1e3:7.1f} us")
            for _ in range(3):
                torch_ref(pred[:1], gt[:1], cut)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(10):
                torch_ref(pred[:1], gt[:1], cut)
            torch.cuda.synchronize()
            line += f"  | torch ops + autograd, 1 image: {(time.perf_counter() - t0) / 10 * 1e6:7.1f} us"
            print(line, flush=True)


if __name__ == "__main__":
    main()
