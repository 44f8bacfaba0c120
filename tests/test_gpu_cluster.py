"""The clustering kernels (esac_b200/csrc/cluster.cu) and the host driver (esac_b200/cluster.py) held to
oracle/cluster_oracle.py, and on the golden fixtures to the reference route (torch + cv2.kmeans)."""
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.cluster import cluster_environment
from esac_b200.compat import SyntheticClusterDataset
from esac_b200.evaluate import PoseEvaluator
from oracle import cluster_oracle as co

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "cluster"


def ragged_maps():
    rng = np.random.default_rng(21)
    maps = []
    for H, W in [(1, 1), (60, 80), (80, 60), (60, 107), (480, 640), (7, 3)]:
        m = (rng.normal(0, 30, (3, H, W)) + rng.uniform(-500, 500, (3, 1, 1))).astype(np.float32)
        m[:, rng.random((H, W)) < 0.5] = 0.0
        maps.append(m)
    maps[0][:, 0, 0] = (1.5, -2.0, 4.0)                    # 1x1, one valid cell
    m = np.zeros((3, 60, 80), np.float32)                  # no valid cell, one cancelling
    m[:, 3, 4] = (1e8, 1, -1e8)
    maps.append(m)
    m = rng.normal(0, 1, (3, 60, 80)).astype(np.float32)   # NaN (first NaN's payload wins) and inf
    m[1, 10, 10] = np.array([0xffc00123], np.uint32).view(np.float32)[0]
    m[1, 50, 3] = np.nan
    m[0, 1, 1] = np.inf
    maps.append(m)
    m = rng.normal(0, 1, (3, 480, 640)).astype(np.float32)  # more valid cells than shared memory holds, with ties
    m[0] = np.round(m[0] * 4) / 4 + 0.5
    maps.append(m)
    return maps


def check_stats(out, maps):
    med, mean, count, status = (t.cpu().numpy() for t in out)
    for b, m in enumerate(maps):
        omed, omean, ocount, ostatus = co.statistics(m)
        assert count[b] == ocount and status[b] == ostatus, b
        np.testing.assert_array_equal(med[b].view(np.uint32), omed.view(np.uint32), err_msg=f"map {b}")
        if ocount:
            v = m.reshape(3, -1)
            cells = v[:, ((v[0] + v[1]) + v[2]) != 0].astype(np.float64)
            exact = cells.sum(1) / ocount
            ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
            fin = np.isfinite(exact)
            assert (np.abs(mean[b][fin] - exact[fin]) <= ulp[fin]).all(), b
            assert (np.isfinite(mean[b]) == fin).all(), b
        else:
            assert np.isnan(mean[b]).all()


@pytest.mark.parametrize("where", ["host", "device"])
def test_statistics_kernel_matches_the_oracle(where):
    maps = ragged_maps()
    ts = [torch.from_numpy(m) for m in maps]
    if where == "device":
        ts = [t.cuda() for t in ts]
    out = api.cluster_statistics(ts)
    assert out[0].device.type == ("cuda" if where == "device" else "cpu")
    check_stats(out, maps)
    assert [int(s) for s in out[3]] == [0, 0, 0, 0, 0, 0, 1, 2, 0]


def test_list_of_equal_maps_is_bitwise_the_stacked_call():
    rng = np.random.default_rng(4)
    stacked = torch.from_numpy(rng.normal(0, 9, (12, 3, 60, 80)).astype(np.float32)).cuda()
    stacked[:, :, rng.random((60, 80)) < 0.3] = 0
    a = api.cluster_statistics(stacked)
    b = api.cluster_statistics(list(stacked.unbind(0)))
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y)


def kmeans_cases():
    rng = np.random.default_rng(8)
    return {
        "separable": np.concatenate([rng.normal(0, 1, (300, 3)), rng.normal(40, 2, (200, 3))]),
        "overlapping": np.concatenate([rng.normal(0, 3, (400, 3)), rng.normal(2, 3, (350, 3))]),
        "n2": rng.normal(0, 1, (2, 3)),
        "duplicates": np.ones((9, 3)) * 7.5,
        "reseed": np.concatenate([np.zeros((6, 3)), np.ones((1, 3)) * 1e-3]),
        "n50000": rng.normal(0, 10, (50000, 3)) * np.array([3.0, 1.0, 0.2]) + rng.integers(0, 2, (50000, 1)) * 25,
    }


@pytest.mark.parametrize("case", list(kmeans_cases()))
def test_kmeans2_matches_the_oracle(case):
    P = kmeans_cases()[case].astype(np.float32)
    seed = 77
    lab, cen, comp = api.kmeans2(torch.from_numpy(P).cuda(), seed, split=3)
    olab, ocen, ocomp = co.kmeans2(P, seed, split=3)
    np.testing.assert_array_equal(lab.cpu().numpy(), olab)
    np.testing.assert_allclose(cen.cpu().numpy(), ocen, rtol=1e-9, atol=0)
    assert abs(comp - ocomp) <= 1e-9 * abs(ocomp)
    assert set(np.unique(olab)) == {0, 1}
    lab2, cen2, comp2 = api.kmeans2(torch.from_numpy(P).cuda(), seed, split=3)
    assert torch.equal(lab, lab2) and torch.equal(cen.view(torch.int32), cen2.view(torch.int32)) and comp == comp2


@pytest.fixture(scope="module")
def synthetic_maps():
    ds = SyntheticClusterDataset(length=6000, training=False, seed=3)
    return [ds.init_map(i) for i in range(len(ds))]


@pytest.mark.parametrize("K", [2, 10, 20, 50])
def test_cluster_environment_matches_the_oracle(synthetic_maps, K):
    c = cluster_environment(synthetic_maps, K, seed=5)
    o = co.cluster_environment([m.numpy() for m in synthetic_maps], K, seed=5)
    np.testing.assert_array_equal(c.labels.cpu().numpy(), o["labels"])
    np.testing.assert_array_equal(c.medians.cpu().numpy().view(np.uint32), o["medians"].view(np.uint32))
    np.testing.assert_array_equal(c.counts.cpu().numpy(), o["counts"])
    np.testing.assert_allclose(c.cam_centers.cpu().numpy(), o["cam_centers"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(c.cam_sizes.cpu().numpy(), o["cam_sizes"], rtol=1e-6, atol=1e-6)
    # float32 targets against float64: exp of an argument x carries ~x ulp of relative error (x reaches ~20 here)
    np.testing.assert_allclose(c.gating_probs.cpu().numpy(), o["gating_probs"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", ["cluster_k4_ragged", "cluster_k5"])
def test_cluster_environment_gives_the_reference_partitions(name):
    g = np.load(GOLDEN / f"{name}.npz")
    K = int(g["K"])
    maps = [torch.from_numpy(g[f"map_{i}"]).cuda() for i in range(int(g["n_maps"]))]
    c = cluster_environment(maps, K)
    lab, ref = c.labels.cpu().numpy(), g["labels"]
    perm = {}
    for a, b in zip(lab, ref):
        assert perm.setdefault(int(a), int(b)) == int(b), "different partitions"
    assert len(set(perm.values())) == K
    order = [k for k, _ in sorted(perm.items(), key=lambda kv: kv[1])]
    np.testing.assert_allclose(c.cam_centers.cpu().numpy()[order], g["cam_centers"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(c.cam_sizes.cpu().numpy()[order], g["cam_sizes"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(c.gating_probs.cpu().numpy()[:, order], g["gating_probs"], rtol=0, atol=1e-5)


def test_cluster_environment_names_the_images_it_cannot_cluster():
    maps = [torch.zeros(3, 6, 8) for _ in range(4)]
    maps[1][:, 2, 2] = 1.0
    with pytest.raises(RuntimeError, match=r"3 image\(s\) cannot be clustered: 0 \(no valid cell\), 2"):
        cluster_environment(maps, 2)
    with pytest.raises(RuntimeError, match=r"num_clusters=5 outside \[1, 4\] for 4 images"):
        cluster_environment([torch.full((3, 2, 2), float(i + 1)) for i in range(4)], 5)


def test_clustered_pose_evaluator_reproduces_the_cluster_mode_table():
    ds = SyntheticClusterDataset(length=40, training=False, seed=2)
    rng = np.random.default_rng(0)
    gt = torch.from_numpy(np.stack([ds.pose(i) for i in range(len(ds))])).cuda()
    est = gt.clone()
    est[:, :3, 3] += torch.from_numpy(rng.normal(0, 0.05, (len(ds), 3)).astype(np.float32)).cuda()
    experts = torch.from_numpy(rng.integers(0, 10, len(ds))).cuda()
    scenes = torch.full((len(ds),), -1, dtype=torch.int64, device="cuda")
    ev = PoseEvaluator(num_scenes=10, capacity=len(ds), clustered=True)
    ev.update(est, gt, experts, scenes)
    t = ev.table(average=False)
    recs = ev.records()
    # test_esac.py in cluster mode: one list, gt_expert = -1 for every image
    r_err, t_err, c_err = list(recs[:, 0]), list(recs[:, 1]), [int(-1) == int(e) for e in recs[:, 4]]
    row = (0, sum(c_err) / len(c_err), sum(1 for r, tt in zip(r_err, t_err) if r < 5 and tt < 5) / len(r_err),
           sorted(r_err)[len(r_err) // 2], sorted(t_err)[len(t_err) // 2])
    assert len(t["rows"]) == 1 and t["excluded"] == 0
    assert t["rows"][0] == row and row[1] == 0
    assert len(t["console"]) == 3
    assert PoseEvaluator(num_scenes=10, capacity=4).clustered is False
