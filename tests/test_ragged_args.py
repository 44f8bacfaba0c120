"""Argument checks of the ragged (list-of-tensors) form of the batched entry points; they run before any CUDA context
exists, so they hold without a GPU."""
import numpy as np
import pytest

from esac_b200.synth import make_scene

SHAPES = [(8, 10), (10, 8), (7, 11)]
B = len(SHAPES)
TAIL = (10.0, 100.0, 0.5, 100.0, 8)
CAMS = ([0] * B, [1] * B, [525.0] * B, [40.0] * B, [32.0] * B)


@pytest.fixture(scope="module")
def batch():
    scenes = [make_scene(E=2, H=h, W=w, M=4, seed=b) for b, (h, w) in enumerate(SHAPES)]
    coords = [s.coords for s in scenes]
    return coords, np.stack([s.assign for s in scenes]), np.stack([s.gt_pose for s in scenes])


def _fwd(coords, assign, poses=None, cams=CAMS):
    import esac_b200.api as api
    poses = np.zeros((len(assign), 4, 4), np.float32) if poses is None else poses
    return api.forward_batch(coords, assign, poses, *cams, *TAIL)


def _bwd(coords, grads, assign, gts, cams=CAMS):
    import esac_b200.api as api
    return api.backward_batch(coords, grads, assign, gts, 1.0, 100.0, 100.0, *cams, *TAIL)


def test_list_lengths_must_match_poses_assignment_and_cameras(batch):
    coords, assign, gts = batch
    with pytest.raises(RuntimeError, match="needs hypAssignment"):
        _fwd(coords, assign[:2])
    with pytest.raises(RuntimeError, match="needs hypAssignment"):
        _fwd(coords, assign, np.zeros((B + 1, 4, 4), np.float32))
    with pytest.raises(RuntimeError, match="focalLength must be"):
        _fwd(coords, assign, cams=CAMS[:2] + ([525.0] * (B - 1),) + CAMS[3:])
    with pytest.raises(RuntimeError, match="gtPoses"):
        _bwd(coords, [np.zeros_like(c) for c in coords], assign, gts[:2])
    with pytest.raises(RuntimeError, match="shiftX must be"):
        _bwd(coords, [np.zeros_like(c) for c in coords], assign, gts, cams=([0] * (B + 1),) + CAMS[1:])
    with pytest.raises(RuntimeError, match="holds 2 tensors for 3 images"):
        _bwd(coords, [np.zeros_like(c) for c in coords[:2]], assign, gts)


def test_mixed_dtype_rank_or_expert_count_is_an_error(batch):
    coords, assign, gts = batch
    with pytest.raises(RuntimeError, match=r"expected scalar type Float but found Double \(sceneCoordinates\[1\]\)"):
        _fwd([coords[0], coords[1].astype(np.float64), coords[2]], assign)
    with pytest.raises(RuntimeError, match=r"expected 4 dims but tensor has 3 \(sceneCoordinates\[2\]\)"):
        _fwd([coords[0], coords[1], coords[2][0]], assign)
    with pytest.raises(RuntimeError, match=r"sceneCoordinates\[1\] must be \[E,3,H,W\] with the E of image 0"):
        _fwd([coords[0], coords[1][:1], coords[2]], assign)
    import esac_b200.api as api
    with pytest.raises(RuntimeError, match=r"prediction\[1\]"):
        api.reproj_loss([coords[0][0], coords[1][0].astype(np.float64)], gts[:2], 525.0, 0, 0, 10.0)
    with pytest.raises(RuntimeError, match=r"expected 3 dims"):
        api.coord_loss([coords[0][0], coords[1]], [coords[0][0], coords[1][0]])


def test_gradient_list_must_match_the_maps(batch):
    import esac_b200.api as api
    coords, assign, gts = batch
    grads = [np.zeros_like(c) for c in coords]
    grads[1] = np.zeros((2, 3, 8, 10), np.float32)
    with pytest.raises(RuntimeError, match=r"outGradients\[1\] is \[2, 3, 8, 10\]"):
        _bwd(coords, grads, assign, gts)
    pred = [c[0] for c in coords]
    og = [np.zeros_like(p) for p in pred]
    og[2] = np.zeros((3, 11, 7), np.float32)
    with pytest.raises(RuntimeError, match=r"outGradients\[2\]"):
        api.reproj_loss(pred, gts, 525.0, 0, 0, 10.0, outGradients=og)
    with pytest.raises(RuntimeError, match=r"outGradients\[2\]"):
        api.coord_loss(pred, pred, outGradients=og)
    # a list of maps needs a list of gradients, and the reverse
    with pytest.raises(RuntimeError, match="outGradients must be a list"):
        _bwd(coords, np.zeros((B, 2, 3, 8, 10), np.float32), assign, gts)


def test_an_empty_list_is_an_error(batch):
    import esac_b200.api as api
    _, assign, gts = batch
    with pytest.raises(RuntimeError, match="empty list"):
        _fwd([], assign[:0])
    with pytest.raises(RuntimeError, match="empty list"):
        _bwd([], [], assign[:0], gts[:0])
    with pytest.raises(RuntimeError, match="empty list"):
        api.reproj_loss([], gts[:0], 525.0, 0, 0, 10.0)
    with pytest.raises(RuntimeError, match="empty list"):
        api.coord_loss([], [])


def test_coordinate_loss_size_difference_of_two_names_the_image():
    import esac_b200.api as api
    pred = [np.ones((3, 8, 10), np.float32), np.ones((3, 12, 9), np.float32)]
    gt = [np.ones((3, 9, 10), np.float32), np.ones((3, 10, 9), np.float32)]
    with pytest.raises(RuntimeError, match="image 1: tensor size mismatch: prediction 12x9, ground truth 10x9"):
        api.coord_loss(pred, gt)
    # both sides are lists
    with pytest.raises(RuntimeError, match="gtCoords must be a list"):
        api.coord_loss(pred, np.ones((2, 3, 8, 10), np.float32))


def test_a_map_too_small_names_the_image(batch):
    coords, assign, gts = batch
    tiny = np.zeros((2, 3, 2, 4), np.float32)   # (W-1)(H-1) = 3 < 4 distinct cells
    with pytest.raises(RuntimeError, match=r"sceneCoordinates\[2\]: map 4x2 too small"):
        _fwd([coords[0], coords[1], tiny], assign)
    with pytest.raises(RuntimeError, match=r"sceneCoordinates\[0\]: map 4x2 too small"):
        _bwd([tiny, coords[1], coords[2]], [np.zeros_like(tiny), np.zeros_like(coords[1]), np.zeros_like(coords[2])], assign, gts)

