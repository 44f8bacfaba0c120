"""Argument errors of api.reproj_loss_async, api.coord_loss_async and api.reserve_loss_async: raised before any context
exists, so they run without a GPU (the tensors here are CPU tensors; the dtype and shape checks come before the device
check)."""
import numpy as np
import pytest
import torch

import esac_b200.api as api


def _reproj_args(B=2, H=6, W=8):
    return dict(prediction=torch.zeros(B, 3, H, W), gtPoses=torch.eye(4).repeat(B, 1, 1),
                shifts=torch.zeros(B, 2, dtype=torch.int32), cameras=torch.ones(B, 3),
                outLosses=torch.zeros(B, dtype=torch.float64), outStatus=torch.zeros(B, dtype=torch.int32),
                outGradients=torch.zeros(B, 3, H, W))


def _reproj(**kw):
    a = _reproj_args(**{k: kw.pop(k) for k in ("B", "H", "W") if k in kw})
    a.update(kw)
    api.reproj_loss_async(a["prediction"], a["gtPoses"], a["shifts"], a["cameras"], 10.0, 8, a["outLosses"], a["outStatus"],
                          outGradients=a["outGradients"])


def _coord_args(B=2, H=6, W=8):
    return dict(prediction=torch.zeros(B, 3, H, W), gtCoords=torch.zeros(B, 3, H, W),
                outLosses=torch.zeros(B, dtype=torch.float64), outGradients=torch.zeros(B, 3, H, W),
                outCounts=torch.zeros(B, dtype=torch.int64))


def _coord(**kw):
    a = _coord_args(**{k: kw.pop(k) for k in ("B", "H", "W") if k in kw})
    a.update(kw)
    api.coord_loss_async(a["prediction"], a["gtCoords"], 10.0, a["outLosses"], outGradients=a["outGradients"],
                         outCounts=a["outCounts"])


def test_cpu_tensors_are_refused_after_the_shape_checks():
    with pytest.raises(RuntimeError, match=r"reproj_loss_async takes CUDA tensors only \(prediction is on the CPU\)"):
        _reproj()
    with pytest.raises(RuntimeError, match=r"coord_loss_async takes CUDA tensors only \(prediction is on the CPU\)"):
        _coord()
    # a ragged list passes the same checks
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \(prediction is on the CPU\)"):
        _reproj(prediction=[torch.zeros(3, 6, 8), torch.zeros(3, 4, 5)], outGradients=None)
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \(prediction is on the CPU\)"):
        _coord(prediction=[torch.zeros(3, 6, 8), torch.zeros(3, 4, 5)], gtCoords=[torch.zeros(3, 6, 8), torch.zeros(3, 5, 5)],
               outGradients=None)


def test_numpy_arrays_are_refused():
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(prediction is a ndarray\)"):
        _reproj(prediction=np.zeros((2, 3, 6, 8), np.float32))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(outStatus is a ndarray\)"):
        _reproj(outStatus=np.zeros(2, np.int32))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(gtCoords\[1\] is a ndarray\)"):
        _coord(prediction=[torch.zeros(3, 6, 8)] * 2, gtCoords=[torch.zeros(3, 6, 8), np.zeros((3, 6, 8), np.float32)],
               outGradients=None)
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(outCounts is a ndarray\)"):
        _coord(outCounts=np.zeros(2, np.int64))


@pytest.mark.parametrize("name,value,msg", [
    ("prediction", torch.zeros(2, 3, 6, 8, dtype=torch.float64), r"expected scalar type Float but found Double \(prediction\)"),
    ("prediction", torch.zeros(3, 6, 8), r"expected 4 dims but tensor has 3 \(prediction\)"),
    ("gtPoses", torch.zeros(2, 4, 4, dtype=torch.float64), r"expected scalar type Float but found Double \(gtPoses\)"),
    ("gtPoses", torch.zeros(4, 4), r"expected 3 dims but tensor has 2 \(gtPoses\)"),
    ("shifts", torch.zeros(2, 2, dtype=torch.int64), r"expected scalar type Int but found Long \(shifts\)"),
    ("cameras", torch.zeros(2, 3, dtype=torch.float64), r"expected scalar type Float but found Double \(cameras\)"),
    ("outLosses", torch.zeros(2), r"expected scalar type Double but found Float \(outLosses\)"),
    ("outStatus", torch.zeros(2, dtype=torch.int64), r"expected scalar type Int but found Long \(outStatus\)"),
    ("outStatus", torch.zeros(2, 1, dtype=torch.int32), r"expected 1 dims but tensor has 2 \(outStatus\)"),
    ("outGradients", torch.zeros(2, 3, 6, 8, dtype=torch.float64), r"Float but found Double \(outGradients\)"),
])
def test_reproj_dtype_and_rank(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _reproj(**{name: value})


@pytest.mark.parametrize("name,value,msg", [
    ("gtPoses", torch.zeros(3, 4, 4), r"gtPoses must be a contiguous \[2, 4, 4\]"),
    ("gtPoses", torch.zeros(2, 4, 4).transpose(1, 2), r"gtPoses must be a contiguous \[2, 4, 4\]"),
    ("shifts", torch.zeros(2, 3, dtype=torch.int32), r"shifts must be a contiguous \[2, 2\]"),
    ("cameras", torch.zeros(3, 2).t(), r"cameras must be a contiguous \[2, 3\]"),
    ("outLosses", torch.zeros(3, dtype=torch.float64), r"outLosses must be a contiguous \[2\]"),
    ("outStatus", torch.zeros(4, dtype=torch.int32)[::2], r"outStatus must be a contiguous \[2\]"),
    ("prediction", torch.zeros(2, 4, 6, 8), r"shapes must be \[B,3,H,W\]"),
    ("prediction", torch.zeros(2, 3, 8, 6).transpose(2, 3), "prediction must be contiguous"),
    ("outGradients", torch.zeros(2, 3, 8, 6).transpose(2, 3), "outGradients must be contiguous"),
    ("outGradients", torch.zeros(2, 3, 6, 7), "outGradients are not of the shape of prediction"),
    ("outGradients", torch.zeros(3, 3, 6, 8), "outGradients holds 3 images for 2 images"),
    ("outGradients", [torch.zeros(3, 6, 8)] * 2, "outGradients must be one stacked tensor"),
])
def test_reproj_shapes_and_layouts(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _reproj(**{name: value})


@pytest.mark.parametrize("name,value,msg", [
    ("prediction", torch.zeros(2, 3, 6, 8, dtype=torch.float16), r"expected scalar type Float but found Half \(prediction\)"),
    ("gtCoords", torch.zeros(2, 3, 6, 8, dtype=torch.float64), r"expected scalar type Float but found Double \(gtCoords\)"),
    ("gtCoords", torch.zeros(3, 6, 8), r"expected 4 dims but tensor has 3 \(gtCoords\)"),
    ("outLosses", torch.zeros(2, dtype=torch.float32), r"expected scalar type Double but found Float \(outLosses\)"),
    ("outCounts", torch.zeros(2, dtype=torch.int32), r"expected scalar type Long but found Int \(outCounts\)"),
    ("outGradients", torch.zeros(2, 3, 6, 8, dtype=torch.float64), r"Float but found Double \(outGradients\)"),
])
def test_coord_dtype_and_rank(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _coord(**{name: value})


@pytest.mark.parametrize("name,value,msg", [
    ("gtCoords", torch.zeros(2, 3, 8, 8), r"image 0: tensor size mismatch: prediction 6x8, ground truth 8x8"),
    ("gtCoords", torch.zeros(3, 3, 6, 8), "gtCoords holds 3 images for 2 images"),
    ("gtCoords", [torch.zeros(3, 6, 8)] * 2, "gtCoords must be one stacked tensor"),
    ("gtCoords", torch.zeros(2, 3, 8, 6).transpose(2, 3), "gtCoords must be contiguous"),
    ("outLosses", torch.zeros(2, 1, dtype=torch.float64), r"expected 1 dims but tensor has 2 \(outLosses\)"),
    ("outLosses", torch.zeros(1, dtype=torch.float64), r"outLosses must be a contiguous \[2\]"),
    ("outCounts", torch.zeros(4, dtype=torch.int64)[::2], r"outCounts must be a contiguous \[2\]"),
    ("outGradients", torch.zeros(2, 3, 7, 8), "outGradients are not of the shape of prediction"),
])
def test_coord_shapes_and_layouts(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _coord(**{name: value})


def test_one_cell_apart_passes_the_shape_checks():
    # util.assert_size tolerates one cell: the device check is what fails
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        _coord(gtCoords=torch.zeros(2, 3, 5, 9))


def test_optional_outputs():
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        _reproj(outGradients=None)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        _coord(outGradients=None, outCounts=None)


def test_empty_batches():
    with pytest.raises(RuntimeError, match="prediction is an empty batch"):
        _reproj(B=0)
    with pytest.raises(RuntimeError, match="prediction is an empty list"):
        _coord(prediction=[], gtCoords=[], outGradients=None)


@pytest.mark.parametrize("sizes", [(0, 6, 8), (1, 0, 8), (1, 6, -1)])
def test_reserve_sizes(sizes):
    with pytest.raises(RuntimeError, match="reserve_loss_async: sizes must be positive"):
        api.reserve_loss_async(*sizes)

