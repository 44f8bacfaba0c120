"""The clustering oracle (oracle/cluster_oracle.py) held to the reference's own route: torch's statistics, the reference's
float32 target sequence, and on the golden fixtures (tests/golden/make_cluster_golden.py: torch + cv2.kmeans) the whole
hierarchy.  CPU only."""
import math
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import cluster_oracle as co

GOLDEN = Path(__file__).resolve().parent / "golden" / "cluster"


def torch_statistics(m):
    """cluster_dataset.py:52-58 and 121-124."""
    d = torch.from_numpy(np.ascontiguousarray(m)).view(3, -1)
    mask = d.sum(0) != 0
    d = d[:, mask]
    return d.median(1)[0].numpy(), (d.sum(1) / mask.sum()).numpy(), int(mask.sum())


def torch_targets(means, centres, sizes, softness=5.0):
    """cluster_dataset.py:222-240, float32."""
    means, centres, sizes = (torch.from_numpy(np.asarray(a, np.float32)) for a in (means, centres, sizes))
    out = torch.zeros(len(means), len(centres))
    for i in range(len(means)):
        d = means[i].unsqueeze(0).expand(centres.size()) - centres
        d = d.norm(dim=1) ** 2
        d = d / sizes[:, 0] / 2
        d = torch.exp(-d * softness)
        d /= torch.sqrt(2 * math.pi * sizes[:, 0])
        d /= d.sum() + 0.0000001
        out[i] = d
    return out.numpy()


def stat_maps():
    rng = np.random.default_rng(5)
    maps = []
    for H, W in [(1, 1), (6, 8), (8, 6), (6, 11), (7, 13), (30, 40)]:
        m = (rng.normal(0, 50, (3, H, W)) + rng.uniform(-300, 300, (3, 1, 1))).astype(np.float32)
        m[:, rng.random((H, W)) < 0.4] = 0.0
        maps.append(m)
    m = rng.normal(0, 1, (3, 6, 8)).astype(np.float32)
    m[:, 0, 0] = (1e8, 1, -1e8)          # cancels: invalid
    m[:, 0, 1] = (1e8, -1e8, 1)          # valid
    m[:, 0, 2] = (2.0, -1.0, -1.0)       # exact zero sum: invalid
    maps.append(m)
    m = rng.normal(0, 1, (3, 5, 9)).astype(np.float32)
    m[1, 2, 3] = np.array([0x7fc00001], np.uint32).view(np.float32)[0]
    m[1, 4, 4] = np.array([0xffc00002], np.uint32).view(np.float32)[0]
    m[2, 0, 1] = np.inf
    maps.append(m)
    one = np.zeros((3, 4, 4), np.float32)
    one[:, 2, 1] = (3.0, -4.0, 5.0)      # one valid cell
    maps.append(one)
    return maps


@pytest.mark.parametrize("i", range(len(stat_maps())))
def test_statistics_match_torch(i):
    m = stat_maps()[i]
    med, mean, count, status = co.statistics(m)
    tmed, tmean, tcount = torch_statistics(m)
    assert count == tcount
    np.testing.assert_array_equal(med.view(np.uint32), tmed.view(np.uint32))      # bitwise, NaN payload included
    np.testing.assert_allclose(mean, tmean, rtol=1e-6, atol=0)
    assert status == (co.STATUS_OK if np.isfinite(med).all() and np.isfinite(mean).all() else co.STATUS_NONFINITE)


def test_statistics_of_a_map_without_ground_truth():
    m = np.zeros((3, 6, 8), np.float32)
    m[:, 1, 1] = (1.0, 1.0, -2.0)
    med, mean, count, status = co.statistics(m)
    assert count == 0 and status == co.STATUS_EMPTY and np.isnan(med).all() and np.isnan(mean).all()


def test_targets_match_the_reference_float32_sequence():
    rng = np.random.default_rng(11)
    K, N = 7, 300
    centres_true = rng.uniform(-200, 200, (K, 3))
    labels = np.arange(N) % K
    means = (centres_true[labels] + rng.normal(0, 8, (N, 3))).astype(np.float32)
    centres, sizes, probs = co.targets(means, labels, K)
    ref = torch_targets(means, centres.astype(np.float32), sizes.astype(np.float32))
    np.testing.assert_allclose(probs, ref, rtol=0, atol=1e-6)


def test_tree_sum_is_a_sum():
    v = np.random.default_rng(2).random(1000)
    total, part = co.tree_sum(v)
    assert part.shape == (co.T,)
    assert abs(total - v.sum()) <= 1e-12 * v.sum()


def test_kmeans_splits_separable_clouds_and_keeps_both_clusters():
    rng = np.random.default_rng(3)
    P = np.concatenate([rng.normal(0, 1, (40, 3)), rng.normal(50, 1, (25, 3))]).astype(np.float32)
    lab, centres, comp = co.kmeans2(P, seed=9)
    assert len(set(lab[:40])) == 1 and len(set(lab[40:])) == 1 and lab[0] != lab[40]
    dup = np.ones((5, 3), np.float32)
    lab, _, comp = co.kmeans2(dup, seed=1)
    assert sorted(np.bincount(lab, minlength=2)) == [1, 4] and comp == 0


def matched(labels, ref_labels, K):
    """The permutation perm (ours -> reference) under which two labelings are the same partition, or None."""
    perm = {}
    for a, b in zip(labels, ref_labels):
        if perm.setdefault(int(a), int(b)) != int(b):
            return None
    return perm if len(set(perm.values())) == K else None


@pytest.mark.parametrize("name", ["cluster_k4_ragged", "cluster_k5"])
def test_oracle_hierarchy_gives_the_reference_partitions(name):
    g = np.load(GOLDEN / f"{name}.npz")
    K = int(g["K"])
    maps = [g[f"map_{i}"] for i in range(int(g["n_maps"]))]
    out = co.cluster_environment(maps, K)
    np.testing.assert_array_equal(out["medians"].view(np.uint32), g["medians"].view(np.uint32))
    np.testing.assert_allclose(out["means"], g["means"], rtol=1e-6, atol=1e-5)   # torch sums in float32
    perm = matched(out["labels"], g["labels"], K)
    assert perm is not None, "different partitions"
    order = [k for k, _ in sorted(perm.items(), key=lambda kv: kv[1])]   # reference cluster j = our cluster order[j]
    np.testing.assert_allclose(out["cam_centers"][order], g["cam_centers"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out["cam_sizes"][order], g["cam_sizes"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out["gating_probs"][:, order], g["gating_probs"], rtol=0, atol=1e-5)


def test_clustered_table_counts_every_image_in_one_row():
    from esac_b200.evaluate import _table
    recs = np.zeros((5, 14))
    recs[:, 0] = [1.0, 9.0, 2.0, 3.0, 0.5]     # rotation errors
    recs[:, 1] = [1.0, 1.0, 7.0, 2.0, 100.0]   # translation errors
    recs[:, 3] = -1                            # scene: none
    recs[:, 4] = [0, 3, 1, 2, 0]
    recs[3, 5] = 1                             # a failed forward stays out
    t = _table(recs, 4, 5, 5, average=False, clustered=True)
    assert t["rows"] == [(0, 0.0, 0.25, 2.0, 7.0)] and t["excluded"] == 1
    assert _table(recs, 4, 5, 5, average=False)["excluded"] == 5
