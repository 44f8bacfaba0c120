"""init_gating.py -c (code/init_gating.py:43-54, 93): initialise the gating network of a clustered environment by the KL
divergence of its output to the soft gating targets of the clustering, on a SyntheticClusterDataset whose clustering
runs on the device (esac_b200.cluster.cluster_environment) when the dataset is built.

    python examples/init_gating_clustered_synthetic.py --images 400 --clusters 10 --iterations 50 --check

--check recomputes the clustering with the float64 restatement in oracle/cluster_oracle.py and compares the labels
(exactly) and the centres, sizes and targets.
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
import torch.optim as optim

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from esac_b200.compat import OUTPUT_SUBSAMPLE, SyntheticClusterDataset, random_shift  # noqa: E402
from train_step_synthetic import TinyGating  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=400)
    ap.add_argument("--clusters", "-c", type=int, default=10)
    ap.add_argument("--iterations", type=int, default=50)
    ap.add_argument("--learningrate", "-lr", type=float, default=0.0001)   # init_gating.py:20
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--check", action="store_true", help="compare the clustering with oracle/cluster_oracle.py")
    opt = ap.parse_args(argv)
    torch.manual_seed(opt.seed)

    t0 = time.time()
    trainset = SyntheticClusterDataset(num_clusters=opt.clusters, length=opt.images, seed=opt.seed)
    torch.cuda.synchronize()
    print(f"Clustered {opt.images} images into {opt.clusters} experts in {time.time() - t0:.2f}s (sizes "
          f"{np.bincount(trainset.labels.cpu().numpy(), minlength=opt.clusters).tolist()})")
    if opt.check:
        from oracle import cluster_oracle as co
        o = co.cluster_environment([trainset.init_map(i).numpy() for i in range(opt.images)], opt.clusters,
                                   softness=trainset.softness, seed=opt.seed)
        assert np.array_equal(trainset.labels.cpu().numpy(), o["labels"]), "labels differ from the oracle"
        for name, ref, tol in (("cam_centers", o["cam_centers"], 1e-6), ("cam_sizes", o["cam_sizes"], 1e-6)):
            err = np.abs(getattr(trainset, name).cpu().numpy() - ref) / np.maximum(np.abs(ref), 1)
            assert err.max() <= tol, f"{name}: {err.max()}"
        dp = np.abs(trainset.gating_probs.cpu().numpy() - o["gating_probs"]).max()
        assert dp <= 1e-6, f"gating_probs: {dp}"
        print(f"check: labels equal, gating_probs within {dp:.2e} of the oracle")

    loader = torch.utils.data.DataLoader(trainset, shuffle=True, batch_size=1)
    model = TinyGating(trainset.num_experts).cuda()
    optimizer = optim.Adam(model.parameters(), lr=opt.learningrate)
    gating_loss = nn.KLDivLoss(reduction="batchmean")
    iteration = 0
    while iteration < opt.iterations:
        for idx, image, focallength, gt_pose, gt_coords, gt_expert in loader:
            image = image.cuda()
            padX, padY, image = random_shift(image, OUTPUT_SUBSAMPLE / 2)
            gating = model(image)
            loss = gating_loss(gating, trainset.gating_probs[idx.cuda()])
            loss.backward()
            optimizer.step()
            optimizer.zero_grad()
            if iteration % 10 == 0:
                print("Iteration: %6d, Gating Loss: %.2f" % (iteration, loss.item()), flush=True)
            iteration += 1
            if iteration >= opt.iterations:
                break
    assert torch.isfinite(loss), "non-finite gating loss"


if __name__ == "__main__":
    main()
