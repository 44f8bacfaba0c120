"""Argument errors of api.hypotheses_forward_async / hypotheses_backward_async / pose_loss_async and of
autograd.esac_hypotheses_async: raised before any context exists, so they run without a GPU (the tensors here are CPU
tensors; the dtype, shape, layout and tape-size checks come before the device check)."""
import numpy as np
import pytest
import torch

import esac_b200.api as api

TAIL = (10.0, 100.0, 0.5, 100.0, 8)   # tau, alpha, beta, maxReproj, sub
E, H, W, M = 3, 6, 8, 16


def _stride():
    return api.hypotheses_tape_stride(E, H, W, M)


def _fwd(B=2, **kw):
    lead = (B,) if B else ()
    a = dict(sceneCoordinates=torch.zeros(lead + (E, 3, H, W)), hypAssignment=torch.zeros(lead + (M,), dtype=torch.int64),
             shifts=torch.zeros(lead + (2,), dtype=torch.int32), cameras=torch.ones(lead + (3,)),
             tapes=torch.zeros(max(B, 1) * _stride(), dtype=torch.uint8), outScores=torch.zeros(lead + (M,), dtype=torch.float64),
             outPoses=torch.zeros(lead + (M, 6), dtype=torch.float64), outContributing=torch.zeros(lead + (M,), dtype=torch.bool),
             outStatus=torch.zeros(lead, dtype=torch.int32))
    a.update(kw)
    api.hypotheses_forward_async(a["sceneCoordinates"], a["hypAssignment"], a["shifts"], a["cameras"], *TAIL, a["tapes"],
                                 a["outScores"], a["outPoses"], a["outContributing"], a["outStatus"])


def _bwd(B=2, **kw):
    lead = (B,) if B else ()
    a = dict(tapes=torch.zeros(max(B, 1) * _stride(), dtype=torch.uint8), sceneCoordinates=torch.zeros(lead + (E, 3, H, W)),
             outGradients=torch.zeros(lead + (E, 3, H, W)), M=M, gradScores=torch.zeros(lead + (M,), dtype=torch.float64),
             gradPoses=torch.zeros(lead + (M, 6), dtype=torch.float64), outStatus=torch.zeros(lead, dtype=torch.int32))
    a.update(kw)
    api.hypotheses_backward_async(a["tapes"], a["sceneCoordinates"], a["outGradients"], a["M"], a["gradScores"],
                                  a["gradPoses"], a["outStatus"])


def _loss(**kw):
    a = dict(poses=torch.zeros(2, M, 6, dtype=torch.float64), gtPose=torch.eye(4).repeat(2, 1, 1))
    a.update(kw)
    api.pose_loss_async(a["poses"], a["gtPose"], 1.0, 100.0, 100.0)


@pytest.mark.parametrize("B", [0, 2])
def test_cpu_tensors_are_refused_after_the_other_checks(B):
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \(sceneCoordinates is on the CPU\)"):
        _fwd(B)
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \((tapes|sceneCoordinates) is on the CPU\)"):
        _bwd(B)
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \(poses is on the CPU\)"):
        _loss()


def test_numpy_arrays_are_refused():
    with pytest.raises(RuntimeError, match="torch CUDA tensors only"):
        _fwd(sceneCoordinates=np.zeros((2, E, 3, H, W), np.float32))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(tapes"):
        _fwd(tapes=np.zeros(2 * _stride(), np.uint8))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(outStatus"):
        _fwd(outStatus=np.zeros(2, np.int32))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(tapes"):
        _bwd(tapes=np.zeros(2 * _stride(), np.uint8))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(gradScores"):
        _bwd(gradScores=np.zeros((2, M)))
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(poses"):
        _loss(poses=np.zeros((2, M, 6)))


@pytest.mark.parametrize("name,value,msg", [
    ("sceneCoordinates", torch.zeros(2, E, 3, H, W, dtype=torch.float64), "expected scalar type Float but found Double"),
    ("hypAssignment", torch.zeros(2, M, dtype=torch.int32), "expected scalar type Long but found Int"),
    ("shifts", torch.zeros(2, 2, dtype=torch.int64), r"\(shifts\)"),
    ("cameras", torch.zeros(2, 3, dtype=torch.float64), r"\(cameras\)"),
    ("outScores", torch.zeros(2, M), r"expected scalar type Double but found Float \(outScores\)"),
    ("outPoses", torch.zeros(2, M, 6), r"\(outPoses\)"),
    ("outContributing", torch.zeros(2, M, dtype=torch.uint8), r"expected scalar type Bool but found Byte \(outContributing\)"),
    ("outStatus", torch.zeros(2, dtype=torch.int64), r"\(outStatus\)"),
    ("tapes", torch.zeros(2 * 4096, dtype=torch.int8), "tapes must be a contiguous 1-D uint8"),
    ("tapes", torch.zeros(2, 4096, dtype=torch.uint8), "tapes must be a contiguous 1-D uint8"),
    ("outScores", torch.zeros(3, M, dtype=torch.float64), r"outScores must be a contiguous \[2, 16\]"),
    ("outPoses", torch.zeros(2, M, 7, dtype=torch.float64), r"outPoses must be a contiguous \[2, 16, 6\]"),
    ("shifts", torch.zeros(2, 3, dtype=torch.int32), r"shifts must be \[2, 2\]"),
])
def test_forward_dtypes_and_shapes(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _fwd(**{name: value})


@pytest.mark.parametrize("name,value,msg", [
    ("sceneCoordinates", torch.zeros(2, E, 3, H, W, dtype=torch.float64), "expected scalar type Float but found Double"),
    ("outGradients", torch.zeros(2, E, 3, H, W + 1), r"outGradients must be a contiguous \[2, 3, 3, 6, 8\]"),
    ("gradScores", torch.zeros(2, M), r"expected scalar type Double but found Float \(gradScores\)"),
    ("gradScores", torch.zeros(2, M + 1, dtype=torch.float64), r"gradScores must be a contiguous \[2, 16\]"),
    ("gradPoses", torch.zeros(2, M, 5, dtype=torch.float64), r"gradPoses must be a contiguous \[2, 16, 6\]"),
    ("outStatus", torch.zeros(2, dtype=torch.int64), r"\(outStatus\)"),
    ("M", 0, "M >= 1"),
])
def test_backward_dtypes_and_shapes(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _bwd(**{name: value})


def test_tapes_too_small_for_the_batch():
    with pytest.raises(RuntimeError, match=r"tapes hold \d+ bytes, 2 image\(s\)"):
        _fwd(tapes=torch.zeros(2 * _stride() - 1, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match=r"tapes hold \d+ bytes, 2 image\(s\)"):
        _bwd(tapes=torch.zeros(_stride(), dtype=torch.uint8))
    # the stride is the tape rounded up to 256 bytes, so one image's bytes do not suffice for two
    assert _stride() % 256 == 0 and _stride() >= api.hypotheses_tape_bytes(E, H, W, M)


def test_non_contiguous_inputs():
    coords = torch.zeros(2, E, 3, H, 2 * W)[..., ::2]
    with pytest.raises(RuntimeError, match="sceneCoordinates must be contiguous"):
        _fwd(sceneCoordinates=coords)
    with pytest.raises(RuntimeError, match="sceneCoordinates must be contiguous"):
        _bwd(sceneCoordinates=coords)
    with pytest.raises(RuntimeError, match="outScores must be a contiguous"):
        _fwd(outScores=torch.zeros(2, 2 * M, dtype=torch.float64)[:, ::2])
    with pytest.raises(RuntimeError, match="gradPoses must be a contiguous"):
        _bwd(gradPoses=torch.zeros(2, 6, M, dtype=torch.float64).transpose(1, 2))
    with pytest.raises(RuntimeError, match="poses must be contiguous"):
        _loss(poses=torch.zeros(2, 6, M, dtype=torch.float64).transpose(1, 2))


def test_row_strided_assignments():
    assign = torch.zeros(2, 2 * M, dtype=torch.int64)[:, :M]
    with pytest.raises(RuntimeError, match="hypAssignment must hold its rows back to back"):
        _fwd(hypAssignment=assign)


def test_pose_loss_async_shapes():
    with pytest.raises(RuntimeError, match=r"gtPose must be a contiguous \[2, 4, 4\]"):
        _loss(gtPose=torch.eye(4).repeat(3, 1, 1))
    with pytest.raises(RuntimeError, match="expected scalar type Double"):
        _loss(poses=torch.zeros(2, M, 6))
    with pytest.raises(RuntimeError, match=r"poses must be \[B, M, 6\]"):
        _loss(poses=torch.zeros(2, M, 5, dtype=torch.float64))


def test_esac_hypotheses_async_refuses_cpu_tensors():
    from esac_b200.autograd import esac_hypotheses_async
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        esac_hypotheses_async(torch.zeros(E, 3, H, W), torch.zeros(M, dtype=torch.int64), torch.zeros(2, dtype=torch.int32),
                              torch.ones(3), *TAIL)
