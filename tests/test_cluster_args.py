"""Argument errors of the clustering calls (api.cluster_statistics, api.kmeans2, api.cluster_targets and their C entry
points): the Python checks raise before any context exists, so all of this runs without a GPU (CPU tensors here; the
dtype, shape and value checks come before the device check)."""
import numpy as np
import pytest
import torch

import esac_b200.api as api


def test_c_entries_refuse_null_handles(lib):
    assert lib.esacb200_cluster_stats_ragged(None, 1, None, None, None, None, None, None, None) == -2
    assert lib.esacb200_kmeans2(None, 2, None, 0, 0, 1, 1, 0.1, None, None, None) == -2
    assert lib.esacb200_cluster_targets(None, 1, None, None, 1, 5.0, None, None, None) == -2


@pytest.mark.parametrize("maps, match", [
    ([], "init_maps is an empty list"),
    (torch.zeros(0, 3, 4, 4), "init_maps is an empty batch"),
    (torch.zeros(2, 4, 4, 4), r"init_maps\[0\] is \[4, 4, 4\]"),
    ([torch.zeros(3, 4, 4), torch.zeros(3, 4, 4, dtype=torch.float64)], "found Double"),
    (torch.zeros(2, 3, 4), "expected 4 dims"),
])
def test_statistics_refuse_before_any_context(maps, match):
    with pytest.raises(RuntimeError, match=match):
        api.cluster_statistics(maps)
    assert not api._contexts


KMEANS_BAD = [
    (dict(points=torch.zeros(1, 3)), "1 points, need at least 2"),
    (dict(points=torch.zeros(5, 2)), r"contiguous \[n,3\]"),
    (dict(points=torch.zeros(5, 3, dtype=torch.float64)), "found Double"),
    (dict(points=np.zeros((5, 3), np.float32)), "takes torch CUDA tensors only"),
    (dict(attempts=0), r"attempts=0 outside \[1, 4096\]"),
    (dict(max_iter=0), "max_iter=0, need at least 1"),
    (dict(eps=-0.1), "need eps >= 0"),
    (dict(eps=float("nan")), "need eps >= 0"),
    (dict(split=-1), "must not be negative"),
    (dict(), r"kmeans2 takes CUDA tensors only \(points is on the CPU\)"),
]


@pytest.mark.parametrize("change, match", KMEANS_BAD, ids=[str(i) for i in range(len(KMEANS_BAD))])
def test_kmeans2_refuses_before_any_context(change, match):
    a = dict(points=torch.zeros(5, 3), seed=0)
    a.update(change)
    with pytest.raises(RuntimeError, match=match):
        api.kmeans2(**a)
    assert not api._contexts


TARGETS_BAD = [
    (dict(labels=torch.tensor([0, 1, 3, 2])), r"label 3 of image 2 outside \[0, 3\)"),
    (dict(labels=torch.tensor([0, -1, 1, 2])), r"label -1 of image 1 outside"),
    (dict(labels=torch.tensor([0, 0, 2, 2])), "cluster 1 has no image"),
    (dict(K=0), r"K=0 outside \[1, 1024\]"),
    (dict(K=1025), r"K=1025 outside"),
    (dict(softness=0.0), "need softness > 0"),
    (dict(softness=-1.0), "need softness > 0"),
    (dict(means=torch.zeros(4, 2)), r"contiguous \[N,3\]"),
    (dict(means=torch.zeros(4, 3, dtype=torch.float64)), "found Double"),
    (dict(labels=torch.tensor([0, 1, 2], dtype=torch.int64)), r"labels must be a contiguous \[4\]"),
    (dict(labels=torch.tensor([0, 1, 2, 1], dtype=torch.int32)), "expected scalar type Long but found Int"),
    (dict(), r"cluster_targets takes CUDA tensors only \(means is on the CPU\)"),
]


@pytest.mark.parametrize("change, match", TARGETS_BAD, ids=[str(i) for i in range(len(TARGETS_BAD))])
def test_cluster_targets_refuse_before_any_context(change, match):
    a = dict(means=torch.zeros(4, 3), labels=torch.tensor([0, 1, 2, 1]), K=3)
    a.update(change)
    with pytest.raises(RuntimeError, match=match):
        api.cluster_targets(**a)
    assert not api._contexts
