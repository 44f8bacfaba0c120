"""Argument errors of api.forward_async / api.reserve_forward_async: raised before any context exists, so they run
without a GPU (the tensors here are CPU tensors; the dtype and shape checks come before the device check)."""
import numpy as np
import pytest
import torch

import esac_b200.api as api

TAIL = (10.0, 100.0, 0.5, 100.0, 8)   # tau, alpha, beta, maxReproj, sub


def _args(B=2, E=3, H=6, W=8, M=16):
    lead = (B,) if B else ()
    return dict(sceneCoordinates=torch.zeros(lead + (E, 3, H, W)), hypAssignment=torch.zeros(lead + (M,), dtype=torch.int64),
                shifts=torch.zeros(lead + (2,), dtype=torch.int32), cameras=torch.ones(lead + (3,)),
                outPoses=torch.zeros(lead + (4, 4)), outExperts=torch.zeros(lead, dtype=torch.int64),
                outStatus=torch.zeros(lead, dtype=torch.int32))


def _call(**kw):
    a = _args(**{k: kw.pop(k) for k in ("B", "E", "H", "W", "M") if k in kw})
    a.update(kw)
    api.forward_async(a["sceneCoordinates"], a["hypAssignment"], a["shifts"], a["cameras"], *TAIL, a["outPoses"],
                      a["outExperts"], a["outStatus"])


@pytest.mark.parametrize("B", [0, 2])
def test_cpu_tensors_are_refused_after_the_shape_checks(B):
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \(sceneCoordinates is on the CPU\)"):
        _call(B=B)


def test_numpy_arrays_are_refused():
    with pytest.raises(RuntimeError, match="torch CUDA tensors only"):
        _call(sceneCoordinates=np.zeros((2, 3, 3, 6, 8), np.float32))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(outStatus"):
        _call(outStatus=np.zeros(2, np.int32))


@pytest.mark.parametrize("name,value,msg", [
    ("sceneCoordinates", torch.zeros(2, 3, 3, 6, 8, dtype=torch.float64), "expected scalar type Float but found Double"),
    ("hypAssignment", torch.zeros(2, 16, dtype=torch.int32), "expected scalar type Long but found Int"),
    ("shifts", torch.zeros(2, 2, dtype=torch.int64), r"expected scalar type Int but found Long \(shifts\)"),
    ("cameras", torch.zeros(2, 3, dtype=torch.float64), r"expected scalar type Float but found Double \(cameras\)"),
    ("outPoses", torch.zeros(2, 4, 4, dtype=torch.float64), r"\(outPoses\)"),
    ("outExperts", torch.zeros(2, dtype=torch.int32), r"expected scalar type Long but found Int \(outExperts\)"),
    ("outStatus", torch.zeros(2, dtype=torch.int64), r"expected scalar type Int but found Long \(outStatus\)"),
    ("hypAssignment", torch.zeros(16, dtype=torch.int64), r"expected 2 dims but tensor has 1 \(hypAssignment\)"),
    ("shifts", torch.zeros(2, dtype=torch.int32), r"expected 2 dims but tensor has 1 \(shifts\)"),
    ("outPoses", torch.zeros(4, 4), r"expected 3 dims but tensor has 2 \(outPoses\)"),
])
def test_dtype_and_rank(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _call(**{name: value})


@pytest.mark.parametrize("name,value,msg", [
    ("hypAssignment", torch.zeros(3, 16, dtype=torch.int64), r"hypAssignment must be \[2, 16\] for 2 image"),
    ("shifts", torch.zeros(2, 3, dtype=torch.int32), r"shifts must be \[2, 2\]"),
    ("cameras", torch.zeros(1, 3), r"cameras must be \[2, 3\]"),
    ("outPoses", torch.zeros(2, 3, 4), r"outPoses must be a contiguous \[2, 4, 4\]"),
    ("outExperts", torch.zeros(3, dtype=torch.int64), r"outExperts must be a contiguous \[2\]"),
    ("outStatus", torch.zeros(4, dtype=torch.int32)[::2], r"outStatus must be a contiguous \[2\]"),
    ("sceneCoordinates", torch.zeros(2, 3, 4, 6, 8), r"must be \[B,E,3,H,W\]"),
    ("sceneCoordinates", torch.zeros(2, 3, 3, 8, 6).transpose(3, 4), "sceneCoordinates must be contiguous"),
    ("cameras", torch.zeros(3, 2).t(), "cameras must be contiguous"),
    ("hypAssignment", torch.zeros(1, 16, dtype=torch.int64).expand(2, 16), "rows back to back"),
])
def test_shapes_and_layouts(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _call(**{name: value})


def test_sizes():
    with pytest.raises(RuntimeError, match="too small to draw 4 distinct cells"):
        _call(H=2, W=3)
    with pytest.raises(RuntimeError, match="no hypothesis"):
        _call(M=0)
    with pytest.raises(RuntimeError, match="no image or no expert"):
        _call(B=2, E=0)


def test_one_image_takes_unbatched_tensors():
    # [E,3,H,W] / [M] / [2] / [3] / [4,4] / [] are one image: the shape checks pass and the device check is what fails
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        _call(B=0)
    with pytest.raises(RuntimeError, match=r"outPoses must be a contiguous \[4, 4\]"):
        _call(B=0, outPoses=torch.zeros(1, 4, 4).view(4, 1, 4)[:, 0].t())
    with pytest.raises(RuntimeError, match=r"expected 0 dims but tensor has 1 \(outExperts\)"):
        _call(B=0, outExperts=torch.zeros(1, dtype=torch.int64))


@pytest.mark.parametrize("sizes", [(0, 1, 6, 8, 16), (1, 1, 6, 8, 0), (1, -1, 6, 8, 16)])
def test_reserve_sizes(sizes):
    with pytest.raises(RuntimeError, match="reserve_forward_async: sizes must be positive"):
        api.reserve_forward_async(*sizes)
