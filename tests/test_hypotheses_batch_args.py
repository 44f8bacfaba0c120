"""The batched hypotheses node without a GPU: argument errors of api.hypotheses_forward_batch / hypotheses_backward_batch
and of the batched api.pose_loss.  Each is raised before any context exists (creating one fails without a GPU, with
another message)."""
import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.synth import make_scene


@pytest.fixture(scope="module")
def batch():
    scenes = [make_scene(E=2, H=8, W=10, M=6, seed=1), make_scene(E=2, H=10, W=8, M=6, seed=2)]
    coords = [s.coords for s in scenes]
    assign = np.stack([s.assign for s in scenes])
    return scenes, coords, assign, scenes[0].params


def test_forward_argument_errors(batch):
    scenes, coords, assign, p = batch
    stacked = np.stack([coords[0], coords[0]])
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.hypotheses_forward_batch(stacked.astype(np.float64), assign, *p)
    with pytest.raises(RuntimeError, match="expected 5 dims"):
        api.hypotheses_forward_batch(coords[0], assign, *p)
    with pytest.raises(RuntimeError, match="expected 4 dims"):
        api.hypotheses_forward_batch([stacked, stacked], assign, *p)
    with pytest.raises(RuntimeError, match="expected scalar type Long but found Int"):
        api.hypotheses_forward_batch(coords, assign.astype(np.int32), *p)
    with pytest.raises(RuntimeError, match="expected 2 dims"):
        api.hypotheses_forward_batch(coords, assign[0], *p)
    with pytest.raises(RuntimeError, match="no hypothesis"):
        api.hypotheses_forward_batch(coords, assign[:, :0], *p)
    with pytest.raises(RuntimeError, match="too small"):
        api.hypotheses_forward_batch([coords[0], np.zeros((2, 3, 2, 3), np.float32)], assign, *p)


def test_forward_batch_size_mismatches(batch):
    scenes, coords, assign, p = batch
    with pytest.raises(RuntimeError, match=r"hypAssignment must be \[2, M\]"):
        api.hypotheses_forward_batch(coords, assign[:1], *p)
    with pytest.raises(RuntimeError, match=r"hypAssignment must be \[3, M\]"):
        api.hypotheses_forward_batch(coords + [coords[0]], assign, *p)
    for i, name in enumerate(("shiftX", "shiftY", "focalLength", "ppointX", "ppointY")):
        q = list(p)
        q[i] = [q[i]] * 3
        with pytest.raises(RuntimeError, match=f"{name} must be"):
            api.hypotheses_forward_batch(coords, assign, *q)


def test_a_list_may_not_mix_experts(batch):
    scenes, coords, assign, p = batch
    with pytest.raises(RuntimeError, match=r"with the E of image 0 \(2\)"):
        api.hypotheses_forward_batch([coords[0], coords[1][:1]], assign, *p)


def _tapes(coords, M):
    return [torch.zeros(api.hypotheses_tape_bytes(c.shape[0], c.shape[2], c.shape[3], M), dtype=torch.uint8) for c in coords]


def test_backward_argument_errors(batch):
    scenes, coords, assign, p = batch
    B, M = assign.shape
    grads = [np.zeros_like(c) for c in coords]
    gs, gp = torch.zeros(B, M, dtype=torch.float64), torch.zeros(B, M, 6, dtype=torch.float64)
    tapes = _tapes(coords, M)
    with pytest.raises(RuntimeError, match=r"tapes\[0\] must be a contiguous CUDA uint8"):
        api.hypotheses_backward_batch(tapes, coords, grads, gs, gp)          # CPU tapes
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.hypotheses_backward_batch(tapes, coords, [g.astype(np.float64) for g in grads], gs, gp)
    with pytest.raises(RuntimeError, match="of sceneCoordinates' kind"):
        api.hypotheses_backward_batch(tapes, coords, np.stack([grads[0], grads[0]]), gs, gp)
    with pytest.raises(RuntimeError, match="outGradients are"):
        api.hypotheses_backward_batch(tapes, coords, grads[::-1], gs, gp)


def test_backward_batch_size_mismatches_and_upstream_shapes(batch, monkeypatch):
    scenes, coords, assign, p = batch
    B, M = assign.shape
    grads = [np.zeros_like(c) for c in coords]
    # CPU stand-ins that pass the tape's kind check, so that the checks behind it are reached
    monkeypatch.setattr(api, "_tape_hypotheses", lambda t, E, H, W, what: t.numel() and M)
    tapes = _tapes(coords, M)
    gs, gp = torch.zeros(B, M, dtype=torch.float64), torch.zeros(B, M, 6, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="outGradients holds 1 tensors for 2 images"):
        api.hypotheses_backward_batch(tapes, coords, grads[:1], gs, gp)
    with pytest.raises(RuntimeError, match="list of 2 tapes"):
        api.hypotheses_backward_batch(tapes[:1], coords, grads, gs, gp)
    with pytest.raises(RuntimeError, match=r"gradScores must be \[2, 6\]"):
        api.hypotheses_backward_batch(tapes, coords, grads, gs[:1], gp)
    with pytest.raises(RuntimeError, match="expected scalar type Double but found Float"):
        api.hypotheses_backward_batch(tapes, coords, grads, gs.float(), gp)
    with pytest.raises(RuntimeError, match="expected 3 dims"):
        api.hypotheses_backward_batch(tapes, coords, grads, gs, gp[0])
    for bad in (gp[:1], gp[:, :-1], gp[..., :3]):
        with pytest.raises(RuntimeError, match=r"gradPoses must be \[2, 6, 6\]"):
            api.hypotheses_backward_batch(tapes, coords, grads, gs, bad)


def test_batched_pose_loss_argument_errors():
    poses = np.zeros((2, 4, 6))
    gts = np.stack([np.eye(4, dtype=np.float32)] * 2)
    with pytest.raises(RuntimeError, match="expected 3 dims but tensor has 2 \\(gtPose\\)"):
        api.pose_loss(poses, gts[0], 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"gtPose must be \[2, 4, 4\]"):
        api.pose_loss(poses, gts[:1], 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"gtPose must be \[2, 4, 4\]"):
        api.pose_loss(poses, gts[:, :3], 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.pose_loss(poses, gts.astype(np.float64), 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"poses must be \[B, M, 6\]"):
        api.pose_loss(poses[..., :3], gts, 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"poses must be \[B, M, 6\]"):
        api.pose_loss(poses[:, :0], gts, 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match="expected scalar type Double but found Float"):
        api.pose_loss(poses.astype(np.float32), gts, 1.0, 100.0, 100.0)
