"""Argument errors of the device-resident image sets (esac_b200.data, api.data_step_async, esacb200_data_step_async): the
Python checks raise before any context exists, so all of this runs without a GPU (the tensors are CPU tensors; the dtype,
shape and contiguity checks come before the device check)."""
import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import data


def test_c_entry_refuses_a_null_handle(lib):
    assert lib.esacb200_data_step_async(None, None, None, None, 1, 0, 1, 1, 0, 0, None, None, 0, None, None, None, 1, None,
                                        1, None, None, None, None, None, None, None, None, None, None) == -2


def _args(B=2, N=3, H=6, W=8, h=2, w=3, capacity=5):
    return dict(pixels=torch.zeros(N * H * W * 3, dtype=torch.uint8), images=torch.zeros(N, 120, dtype=torch.uint8),
                plan=torch.zeros(capacity, 10, dtype=torch.int32), state=torch.zeros(2, dtype=torch.int64), group=0,
                mean=data.ROOM_MEAN, std=data.ROOM_STD, work=torch.zeros(B, dtype=torch.int64),
                outImage=torch.zeros(B, 3, H, W), outShifts=torch.zeros(B, 2, dtype=torch.int32), outCameras=torch.zeros(B, 3),
                outPoses=torch.zeros(B, 4, 4), outScenes=torch.zeros(B, dtype=torch.int64),
                outIndices=torch.zeros(B, dtype=torch.int64), outStatus=torch.zeros(1, dtype=torch.int32),
                gt=torch.zeros(N * 3 * h * w), outCoords=torch.zeros(B, 3, h, w), attachments=[torch.zeros(N, 4)],
                outAttachments=[torch.zeros(B, 4)])


BAD = [
    ("pixels", torch.zeros(10, dtype=torch.int8), "expected scalar type Byte but found Char"),
    ("pixels", torch.zeros(2, 5, dtype=torch.uint8), "expected 1 dims"),
    ("pixels", np.zeros(10, np.uint8), "takes torch tensors only"),
    ("images", torch.zeros(3, 119, dtype=torch.uint8), r"images must be a contiguous \[3, 120\]"),
    ("images", torch.zeros(0, 120, dtype=torch.uint8), "the set holds 0 images"),
    ("plan", torch.zeros(5, 9, dtype=torch.int32), r"plan must be a contiguous \[5, 10\]"),
    ("plan", torch.zeros(0, 10, dtype=torch.int32), "the plan 0 rows"),
    ("plan", torch.zeros(5, 10, dtype=torch.int64), "expected scalar type Int but found Long"),
    ("state", torch.zeros(4, dtype=torch.int64), r"state must be a contiguous \[2\]"),
    ("group", -1, "group must be a non-negative int"),
    ("group", 1.0, "group must be a non-negative int"),
    ("mean", [0.4, 0.4], "mean and std must be three finite numbers"),
    ("std", 0.0, "std nonzero"),
    ("std", float("nan"), "finite"),
    ("work", torch.zeros(3, dtype=torch.int64), r"work must be a contiguous \[2\]"),
    ("outImage", torch.zeros(2, 1, 6, 8), r"outImage must be \[B,3,H,W\]"),
    ("outImage", torch.zeros(2, 3, 6, 8, dtype=torch.float64), "found Double"),
    ("outImage", torch.zeros(0, 3, 6, 8), r"outImage must be \[B,3,H,W\] with B in"),
    ("outImage", torch.zeros(1, 3, 6, 9000), "sides in"),
    ("outShifts", torch.zeros(2, 2, dtype=torch.int64), "expected scalar type Int"),
    ("outCameras", torch.zeros(2, 4), r"outCameras must be a contiguous \[2, 3\]"),
    ("outPoses", torch.zeros(4, 4, 2).permute(2, 0, 1), "must be a contiguous"),
    ("outScenes", torch.zeros(2, dtype=torch.int32), "expected scalar type Long"),
    ("outIndices", torch.zeros(3, dtype=torch.int64), r"outIndices must be a contiguous \[2\]"),
    ("outStatus", torch.zeros(2, dtype=torch.int32), r"outStatus must be a contiguous \[1\]"),
    ("gt", None, "gt and outCoords must both be given"),
    ("outCoords", torch.zeros(2, 2, 2, 3), r"outCoords must be a contiguous \[2, 3, 2, 3\]"),
    ("attachments", [torch.zeros(4, 4)], r"attachments\[0\] must be a contiguous float32 \[3, ...\]"),
    ("attachments", [torch.zeros(3, 4, dtype=torch.float64)], "found Double"),
    ("attachments", [], "0 attachments for 1 outputs"),
    ("outAttachments", [torch.zeros(2, 5)], r"outAttachments\[0\] must be a contiguous \[2, 4\]"),
]


@pytest.mark.parametrize("name, value, match", BAD, ids=[f"{n}-{i}" for i, (n, _, _) in enumerate(BAD)])
def test_step_refuses_before_any_context(name, value, match):
    a = _args()
    a[name] = value
    with pytest.raises(RuntimeError, match=match):
        api.data_step_async(**a)
    assert not api._contexts


def test_step_refuses_cpu_tensors_before_any_context():
    with pytest.raises(RuntimeError, match="pixels must be a CUDA tensor or a pinned CPU tensor"):
        api.data_step_async(**_args())
    assert not api._contexts


def _image(H=6, W=8):
    return np.zeros((H, W, 3), np.uint8)


SET_BAD = [
    (dict(images=[np.zeros((6, 8, 3), np.float32)]), "images must be uint8"),
    (dict(images=[np.zeros((6, 8, 4), np.uint8)]), r"images must be \[H,W,3\] RGB or \[H,W\] gray"),
    (dict(images=[np.zeros((6, 8, 3, 1), np.uint8)]), r"images must be \[H,W,3\]"),
    (dict(images=[np.zeros((1, 9000, 3), np.uint8)]), "has a side above 8192"),
    (dict(images=[]), "at least one image"),
    (dict(poses=np.zeros((2, 4, 4))), r"poses must be \[1,4,4\]"),
    (dict(focal=[500.0, 1.0]), "focal and scenes must hold 1 values"),
    (dict(gt=[torch.zeros(3, 2, 2, dtype=torch.float64)]), r"gt\[0\] must be a float32 \[3,h,w\]"),
    (dict(gt=[torch.zeros(2, 2, 2)]), r"gt\[0\] must be a float32 \[3,h,w\]"),
    (dict(gt=[]), "gt must hold 1 maps"),
    (dict(attachments={"prior": torch.zeros(2, 3)}), r"must be a float32 tensor \[1, ...\]"),
    (dict(attachments={"image": torch.zeros(1, 3)}), "is taken by an output"),
    (dict(mean=[0.4, 0.4]), "mean must be a number or three"),
    (dict(std=0.0), "std must be nonzero"),
    (dict(storage="host"), "storage must be 'device' or 'pinned'"),
    (dict(plan_capacity=0), "plan_capacity must be positive"),
]


@pytest.mark.parametrize("kw, match", SET_BAD, ids=[f"{i}" for i in range(len(SET_BAD))])
def test_set_refuses_before_any_context(kw, match):
    a = dict(images=[_image()], poses=np.eye(4, dtype=np.float32)[None], focal=[500.0], scenes=[0])
    a.update(kw)
    with pytest.raises(ValueError, match=match):
        data.DeviceImageSet(**a)
    assert not api._contexts


def _plan(images, groups, batch=1, ops=None):
    rows = np.zeros(len(images), api.DATA_ROW)
    rows["image"] = images
    if ops is not None:
        rows["n_ops"] = len(ops)
        rows["ops"][:, :len(ops)] = ops
    return data.Plan(rows, groups, batch)


PLAN_BAD = [
    (_plan([0, 1, 2, 0, 1, 2], [0] * 6), 5, "more than the set's plan capacity 5"),
    (_plan([0, 1], [0]), 8, "2 rows for 1 steps of 1"),
    (_plan([0, 3], [0, 0]), 8, r"outside \[0, 3\)"),
    (_plan([0, -1], [0, 0]), 8, r"outside \[0, 3\)"),
    (_plan([0, 2], [0, 0]), 8, "does not hold the shape group"),
    (_plan([0, 1], [0, 0], ops=[0, 0]), 8, "bad jitter"),
    (_plan([0, 1], [0, 0], ops=[3]), 8, "bad jitter"),
]


@pytest.mark.parametrize("plan, capacity, match", PLAN_BAD, ids=[f"{i}" for i in range(len(PLAN_BAD))])
def test_plan_refused(plan, capacity, match):
    with pytest.raises(ValueError, match=match):
        data.check_plan(plan, 3, np.array([0, 0, 1], np.int32), capacity)


def test_hue_refused():
    from torchvision import transforms
    with pytest.raises(ValueError, match="hue jitter is not supported"):
        data.ClusterDraws(4, jitter=transforms.ColorJitter(brightness=0.2, hue=0.1))
    assert not api._contexts
