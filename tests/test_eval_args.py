"""Argument errors of the pose evaluation (api.evaluate_poses, api.evaluate_poses_async, esac_b200.evaluate.PoseEvaluator,
esacb200_eval_poses*): the Python checks raise before any context exists, so all of this runs without a GPU (the tensors
here are CPU tensors; the dtype, shape and contiguity checks come before the device check)."""
import ctypes as C

import pytest
import torch

import esac_b200.api as api
from esac_b200.evaluate import PoseEvaluator


def _args(B=3, E=4, capacity=8):
    return dict(outPoses=torch.zeros(B, 4, 4), gtPoses=torch.zeros(B, 4, 4), experts=torch.zeros(B, dtype=torch.int64),
                gtScenes=torch.zeros(B, dtype=torch.int64), outRecords=torch.zeros(capacity, 14, dtype=torch.float64),
                state=torch.zeros(4, dtype=torch.int64), hist=torch.zeros(B, E), status=torch.zeros(B, dtype=torch.int32))


def test_c_entries_refuse_null_handles(lib):
    for name in ("esacb200_eval_poses", "esacb200_eval_poses_async"):
        assert getattr(lib, name)(None, 1, None, None, None, None, None, 0, None, None, 1, None) == -2


BAD = [
    ("outPoses", torch.zeros(3, 4, 4, dtype=torch.float64), "expected scalar type Float but found Double"),
    ("outPoses", torch.zeros(3, 3, 4), r"outPoses must be \[B,4,4\] or \[4,4\]"),
    ("outPoses", torch.zeros(2, 3, 4, 4), "expected 2 dims"),
    ("outPoses", torch.zeros(0, 4, 4), r"outPoses must be \[B,4,4\]"),
    ("outPoses", [[0.0] * 4] * 4, "takes torch CUDA tensors only"),
    ("gtPoses", torch.zeros(2, 4, 4), r"gtPoses must be a contiguous \[3, 4, 4\]"),
    ("gtPoses", torch.zeros(3, 4, 4).transpose(1, 2), r"gtPoses must be a contiguous"),
    ("gtPoses", torch.zeros(3, 4, 4, dtype=torch.float16), "found Half"),
    ("experts", torch.zeros(3, dtype=torch.int32), "expected scalar type Long but found Int"),
    ("experts", torch.zeros(4, dtype=torch.int64), r"experts must be a contiguous \[3\]"),
    ("gtScenes", torch.zeros(3, 1, dtype=torch.int64), "expected 1 dims"),
    ("gtScenes", 2, "takes torch CUDA tensors only"),
    ("outRecords", torch.zeros(8, 13, dtype=torch.float64), r"outRecords must be a contiguous \[8, 14\]"),
    ("outRecords", torch.zeros(8, 14), "expected scalar type Double but found Float"),
    ("outRecords", torch.zeros(0, 14, dtype=torch.float64), "outRecords holds no row"),
    ("outRecords", torch.zeros(14, 8, dtype=torch.float64).t(), "must be a contiguous"),
    ("state", torch.zeros(3, dtype=torch.int64), r"state must be a contiguous \[4\]"),
    ("state", torch.zeros(4, dtype=torch.int32), "expected scalar type Long"),
    ("hist", torch.zeros(3, 0), r"E=0 experts, outside \[1, 1024\]"),
    ("hist", torch.zeros(3, 1025), r"E=1025 experts, outside \[1, 1024\]"),
    ("hist", torch.zeros(3, 4, 1), r"hist must be a float32 tensor \[B,E\] or \[E\]"),
    ("hist", torch.zeros(2, 4), r"hist must be a contiguous \[3, 4\]"),
    ("hist", torch.zeros(3, 4, dtype=torch.float64), "found Double"),
    ("status", torch.zeros(3, dtype=torch.int64), "expected scalar type Int but found Long"),
    ("status", torch.zeros(2, dtype=torch.int32), r"status must be a contiguous \[2\]|status must be a contiguous \[3\]"),
]


@pytest.mark.parametrize("name, value, match", BAD, ids=[f"{n}-{i}" for i, (n, _, _) in enumerate(BAD)])
def test_async_refuses_before_any_context(name, value, match):
    a = _args()
    a[name] = value
    with pytest.raises(RuntimeError, match=match):
        api.evaluate_poses_async(**a)
    assert not api._contexts


@pytest.mark.parametrize("name, value, match", [b for b in BAD if b[0] not in ("outRecords", "state")],
                         ids=[f"{n}-{i}" for i, (n, _, _) in enumerate(BAD) if n not in ("outRecords", "state")])
def test_eager_refuses_before_any_context(name, value, match):
    a = _args()
    del a["outRecords"], a["state"]
    a[name] = value
    with pytest.raises(RuntimeError, match=match):
        api.evaluate_poses(**a)
    assert not api._contexts


def test_cpu_tensors_are_refused_before_any_context():
    with pytest.raises(RuntimeError, match=r"evaluate_poses_async takes CUDA tensors only \(outPoses is on the CPU\)"):
        api.evaluate_poses_async(**_args())
    a = _args()
    del a["outRecords"], a["state"]
    with pytest.raises(RuntimeError, match=r"evaluate_poses takes CUDA tensors only"):
        api.evaluate_poses(**a)
    one = {k: (v[0] if k in ("outPoses", "gtPoses", "experts", "gtScenes", "hist", "status") else v) for k, v in a.items()}
    with pytest.raises(RuntimeError, match="CUDA tensors only"):   # the [4,4] form passes the shape checks
        api.evaluate_poses(**one)
    assert not api._contexts


@pytest.mark.parametrize("num_scenes, capacity", [(0, 4), (3, 0), (-1, -1)])
def test_evaluator_sizes(num_scenes, capacity):
    with pytest.raises(RuntimeError, match="num_scenes >= 1 and capacity >= 1"):
        PoseEvaluator(num_scenes, capacity, device="cpu")
    assert not api._contexts


def test_evaluator_update_checks_before_any_context():
    ev = PoseEvaluator(3, 4, device="cpu")
    a = _args()
    with pytest.raises(RuntimeError, match="found Double"):
        ev.update(a["outPoses"].double(), a["gtPoses"], a["experts"], a["gtScenes"])
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ev.update(a["outPoses"], a["gtPoses"], a["experts"], a["gtScenes"], hist=a["hist"], status=a["status"])
    assert not api._contexts
