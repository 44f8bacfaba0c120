"""Argument checks of the per-image cameras of the batched entry points; they run before any CUDA context exists, so
they hold without a GPU."""
import ctypes as C

import numpy as np
import pytest

from esac_b200.synth import make_scene

B = 3


@pytest.fixture(scope="module")
def batch():
    scenes = [make_scene(E=2, H=8, W=10, M=4, seed=b) for b in range(B)]
    coords = np.stack([s.coords for s in scenes])
    return coords, np.stack([s.assign for s in scenes]), np.stack([s.gt_pose for s in scenes])


GOOD = {"shiftX": [0] * B, "shiftY": [1] * B, "f": [525.0] * B, "ppx": [40.0] * B, "ppy": [32.0] * B}
BAD = [("shiftX", [0] * (B - 1)), ("shiftY", [0] * (B + 1)), ("f", np.full(B + 1, 525.0)), ("ppx", [40.0] * (B - 1)),
       ("ppy", np.zeros((0,)))]


def _cams(name, value):
    cams = dict(GOOD)
    cams[name] = value
    return cams["shiftX"], cams["shiftY"], cams["f"], cams["ppx"], cams["ppy"]


@pytest.mark.parametrize("name,value", BAD, ids=[n for n, _ in BAD])
def test_forward_batch_rejects_a_camera_array_of_the_wrong_length(batch, name, value):
    import esac_b200.api as api
    coords, assign, _ = batch
    with pytest.raises(RuntimeError, match="must be"):
        api.forward_batch(coords, assign, np.zeros((B, 4, 4), np.float32), *_cams(name, value), 10.0, 100.0, 0.5, 100.0, 8)


@pytest.mark.parametrize("name,value", BAD, ids=[n for n, _ in BAD])
def test_backward_batch_rejects_a_camera_array_of_the_wrong_length(batch, name, value):
    import esac_b200.api as api
    coords, assign, gts = batch
    with pytest.raises(RuntimeError, match="must be"):
        api.backward_batch(coords, np.zeros_like(coords), assign, gts, 1.0, 100.0, 100.0, *_cams(name, value), 10.0, 100.0,
                           0.5, 100.0, 8)


@pytest.mark.parametrize("name,value", BAD, ids=[n for n, _ in BAD])
def test_reproj_loss_rejects_a_camera_array_of_the_wrong_length(batch, name, value):
    import esac_b200.api as api
    coords, _, gts = batch
    sx, sy, f, ppx, ppy = _cams(name, value)
    with pytest.raises(RuntimeError, match="must be"):
        api.reproj_loss(np.ascontiguousarray(coords[:, 0]), gts, f, sx, sy, 10.0, 8, ppx, ppy)


def test_reproj_loss_checks_the_focal_length_against_the_default_principal_point(batch):
    import esac_b200.api as api
    coords, _, gts = batch
    with pytest.raises(RuntimeError, match="focalLength must be"):
        api.reproj_loss(np.ascontiguousarray(coords[:, 0]), gts, [525.0] * (B + 1), 0, 0, 10.0)


def test_per_image_values_round_like_ctypes():
    """A DataLoader hands focal lengths over as a float64 tensor; each value becomes the float32 a Python float would."""
    import torch
    from esac_b200.api import _per_image
    vals = [525.3, 1e-3 + 1 / 3, 2 ** 24 + 1.0, 583.2999999999]
    for v in (vals, np.array(vals), torch.tensor(vals, dtype=torch.float64)):
        got = _per_image(v, len(vals), np.float32, "focalLength")
        assert got.dtype == np.float32 and got.flags["C_CONTIGUOUS"]
        assert [float(x) for x in got] == [C.c_float(x).value for x in vals]
    # a number (also a 0-d tensor, e.g. focallength[0]) is one value for every image
    assert _per_image(torch.tensor(525.3, dtype=torch.float64), 2, np.float32, "f").tolist() == [C.c_float(525.3).value] * 2
    assert _per_image(-3, 2, np.int32, "shiftX").tolist() == [-3, -3]
