"""The hypotheses node without a GPU: argument errors of api.hypotheses_forward / hypotheses_backward / pose_loss (raised
before any context exists), the tape size, and autograd.pose_to_transform against the oracle's pose2trans and gradcheck."""
import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.autograd import pose_to_transform
from esac_b200.synth import make_scene
from oracle import esac_oracle as O


@pytest.fixture(scope="module")
def sc():
    return make_scene(E=2, H=8, W=10, M=6)


def test_forward_argument_errors(sc):
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.hypotheses_forward(sc.coords.astype(np.float64), sc.assign, *sc.params)
    with pytest.raises(RuntimeError, match="expected scalar type Long but found Int"):
        api.hypotheses_forward(sc.coords, sc.assign.astype(np.int32), *sc.params)
    with pytest.raises(RuntimeError, match="expected 4 dims"):
        api.hypotheses_forward(sc.coords[0], sc.assign, *sc.params)
    with pytest.raises(RuntimeError, match=r"\[E, 3, H, W\]"):
        api.hypotheses_forward(np.zeros((2, 4, 8, 10), np.float32), sc.assign, *sc.params)
    with pytest.raises(RuntimeError, match="too small"):
        api.hypotheses_forward(np.zeros((2, 3, 2, 3), np.float32), sc.assign, *sc.params)
    with pytest.raises(RuntimeError, match="no hypothesis"):
        api.hypotheses_forward(sc.coords, sc.assign[:0], *sc.params)


def test_backward_argument_errors(sc):
    M = sc.assign.shape[0]
    E, _, H, W = sc.coords.shape
    tape = torch.zeros(api.hypotheses_tape_bytes(E, H, W, M), dtype=torch.uint8)
    g = np.zeros_like(sc.coords)
    gs, gp = torch.zeros(M, dtype=torch.float64), torch.zeros(M, 6, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="tape must be"):
        api.hypotheses_backward(tape, sc.coords, g, gs, gp)          # a CPU tape
    with pytest.raises(RuntimeError, match="tape must be"):
        api.hypotheses_backward(np.zeros(16, np.uint8), sc.coords, g, gs, gp)
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.hypotheses_backward(tape, sc.coords, g.astype(np.float64), gs, gp)
    with pytest.raises(RuntimeError, match="must both be"):
        api.hypotheses_backward(tape, sc.coords, g[:1], gs, gp)
    with pytest.raises(RuntimeError, match="expected scalar type Double but found Float"):
        api.hypotheses_backward(tape, sc.coords, g, gs.float(), gp)
    with pytest.raises(RuntimeError, match="expected 2 dims"):
        api.hypotheses_backward(tape, sc.coords, g, gs, gp[0])
    with pytest.raises(RuntimeError, match=r"gradPoses must be \[M, 6\]"):
        api.hypotheses_backward(tape, sc.coords, g, gs, gp[:, :3])
    with pytest.raises(RuntimeError, match=r"gradPoses must be \[M, 6\]"):
        api.hypotheses_backward(tape, sc.coords, g, gs[:-1], gp)


def test_pose_loss_argument_errors(sc):
    poses = np.zeros((4, 6))
    with pytest.raises(RuntimeError, match="expected scalar type Double but found Float"):
        api.pose_loss(poses.astype(np.float32), sc.gt_pose, 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.pose_loss(poses, sc.gt_pose.astype(np.float64), 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"poses must be \[M, 6\]"):
        api.pose_loss(np.zeros((4, 3)), sc.gt_pose, 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"poses must be \[M, 6\]"):
        api.pose_loss(np.zeros((0, 6)), sc.gt_pose, 1.0, 100.0, 100.0)
    with pytest.raises(RuntimeError, match=r"gtPose must be \[4, 4\]"):
        api.pose_loss(poses, sc.gt_pose[:3], 1.0, 100.0, 100.0)


def test_tape_size_grows_with_hypotheses_and_cells():
    b = api.hypotheses_tape_bytes
    assert b(3, 48, 64, 48) > 0
    assert b(3, 48, 64, 49) > b(3, 48, 64, 48)
    assert b(3, 48, 65, 48) > b(3, 48, 64, 48)
    assert b(1, 48, 64, 48) == b(7, 48, 64, 48)  # the tape holds per-hypothesis state only
    assert b(0, 48, 64, 48) == 0 and b(3, 48, 64, 0) == 0


def _rvec(rng, angle):
    v = rng.normal(size=3)
    return v / np.linalg.norm(v) * angle


def _poses():
    rng = np.random.default_rng(5)
    rows = [np.r_[_rvec(rng, a), rng.normal(size=3) * 3] for a in (0.0, 1e-9, 1e-5, 1e-3, 0.3, 2.0, np.pi - 1e-6)]
    rows += [np.r_[rng.normal(size=3), rng.normal(size=3)] for _ in range(5)]
    return torch.tensor(np.array(rows))


def test_pose_to_transform_matches_oracle_pose2trans():
    P = _poses()
    T = pose_to_transform(P).numpy()
    for i in range(P.shape[0]):
        ref = O.pose2trans(P[i, :3].numpy(), P[i, 3:].numpy())
        assert np.abs(T[i] - ref).max() < 1e-12, (i, np.abs(T[i] - ref).max())


@pytest.mark.parametrize("angle", [0.0, 1e-9, 1e-3, 0.7, np.pi - 1e-6])
def test_pose_to_transform_gradcheck(angle):
    rng = np.random.default_rng(11)
    p = torch.tensor(np.r_[_rvec(rng, angle), rng.normal(size=3)][None], requires_grad=True)
    assert torch.autograd.gradcheck(pose_to_transform, (p,))
    g, = torch.autograd.grad(pose_to_transform(p).sum(), p)
    assert torch.isfinite(g).all()


def test_pose_to_transform_series_joins_the_closed_form():
    """Just below and above the switch to the series, transform and gradient agree to rounding."""
    d = np.array([0.6, -0.3, 0.74])
    d /= np.linalg.norm(d)
    out = []
    for th in (1e-3 * (1 - 1e-9), 1e-3 * (1 + 1e-9)):
        p = torch.tensor(np.r_[d * th, 1.0, 2.0, 3.0][None], requires_grad=True)
        T = pose_to_transform(p)
        g, = torch.autograd.grad((T * torch.arange(16.0, dtype=T.dtype).reshape(4, 4)).sum(), p)
        out.append((T.detach(), g))
    assert (out[0][0] - out[1][0]).abs().max() < 1e-11
    assert (out[0][1] - out[1][1]).abs().max() < 1e-9
