"""The getters of what the last call left (esacb200_get_hypotheses, esacb200_copy_last_scores, esacb200_get_sample_profile)
read only what that call wrote, and whenever get_hypotheses writes rows it writes exactly stats()["M"] of them, the rows
Context.hypotheses() allocates (run with `-m gpu`).

The cases that end in a failing getter call esacb200_get_hypotheses through ctypes with buffers sized for the one M every
call uses, so that a library which does read stale buffers writes only memory the test owns."""
import numpy as np
import pytest

from esac_b200.synth import make_scene

pytestmark = pytest.mark.gpu

M = 32
W_LOSS = (1.0, 100.0, 100.0)


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


@pytest.fixture(scope="module")
def sc():
    return make_scene(E=2, H=30, W=40, M=M, sub=8, seed=3)


def _get_hypotheses(api, losses=False):
    """esacb200_get_hypotheses into buffers of M rows: its status and the rows."""
    ctx = api.context()
    out = {"poses": np.zeros((M, 6)), "cells": np.zeros((M, 4, 2), np.int32), "tries": np.zeros(M, np.int32),
           "scores": np.zeros(M), "probs": np.zeros(M), "refined": np.zeros((M, 6)), "losses": np.zeros(M)}
    rc = ctx.lib.esacb200_get_hypotheses(ctx.handle, out["poses"].ctypes.data, out["cells"].ctypes.data, out["tries"].ctypes.data,
                                         out["scores"].ctypes.data, out["probs"].ctypes.data, out["refined"].ctypes.data,
                                         out["losses"].ctypes.data if losses else None)
    return rc, out


def _copy_last_scores(api):
    """Context.copy_last_scores into M doubles: the scores, or None where the getter fails."""
    dst = np.zeros(M)
    try:
        api.context().copy_last_scores(dst)
    except RuntimeError:
        return None
    return dst


def _sample_profile(api):
    try:
        return api.context().sample_profile()
    except RuntimeError:
        return None


def _forward(api, sc, seed=7):
    api.set_seed(seed)
    out = np.zeros((4, 4), np.float32)
    api.forward(sc.coords, sc.assign, out, *sc.params)


def _backward(api, sc, seed=7):
    api.set_seed(seed)
    g = np.zeros_like(sc.coords)
    api.backward(sc.coords, g, sc.assign, sc.gt_pose, *W_LOSS, *sc.params)


def _refine_params(sc):
    shiftX, shiftY, f, ppx, ppy, tau, _alpha, _beta, max_reproj, sub = sc.params
    return shiftX, shiftY, f, ppx, ppy, tau, max_reproj, sub


def test_pose_loss_after_forward_leaves_no_hypotheses(api, sc):
    import torch
    _forward(api, sc)
    assert _get_hypotheses(api)[0] == 0
    poses = torch.zeros(M, 6, dtype=torch.float64)
    poses[:, 5] = 1.0
    api.pose_loss(poses, torch.from_numpy(sc.gt_pose), *W_LOSS)
    assert api.last_stats()["M"] == 0
    rc, _ = _get_hypotheses(api)
    assert rc != 0
    assert "left no hypotheses" in api.context().lib.esacb200_last_error(api.context().handle).decode()


def test_hypotheses_backward_leaves_no_hypotheses(api, sc):
    import torch
    api.set_seed(11)
    coords = torch.from_numpy(sc.coords).cuda()
    scores, poses, contrib, tape = api.hypotheses_forward(coords, sc.assign, *sc.params)
    rc, hy = _get_hypotheses(api)
    assert rc == 0 and np.array_equal(hy["scores"], scores.cpu().numpy())
    g = torch.zeros_like(coords)
    api.hypotheses_backward(tape, coords, g, torch.ones(M, dtype=torch.float64, device="cuda"), None)
    torch.cuda.synchronize()
    assert api.last_stats()["M"] == M
    assert _get_hypotheses(api)[0] != 0
    assert _copy_last_scores(api) is None
    assert _sample_profile(api) is None


def test_refine_poses_after_backward_leaves_no_losses_scores_or_profile(api, sc):
    _backward(api, sc)
    rc, hy = _get_hypotheses(api, losses=True)
    assert rc == 0 and np.isfinite(hy["losses"]).all()
    assert _copy_last_scores(api) is not None and _sample_profile(api) is not None
    api.refine_poses(sc.coords, sc.assign, hy["poses"], *_refine_params(sc))
    assert _get_hypotheses(api, losses=True)[0] != 0
    assert _get_hypotheses(api)[0] != 0
    assert _copy_last_scores(api) is None
    assert _sample_profile(api) is None


def test_score_poses_after_forward_leaves_scores_but_no_sampling(api, sc):
    _forward(api, sc)
    rc, hy = _get_hypotheses(api)
    assert rc == 0
    poses = hy["poses"].copy()
    poses[::2, 3:] += 0.05  # not the forward's scores
    scores = api.score_poses(sc.coords, sc.assign, poses, *sc.params)
    got = _copy_last_scores(api)
    assert got is not None and np.array_equal(got, scores) and not np.array_equal(scores, hy["scores"])
    assert _sample_profile(api) is None
    assert _get_hypotheses(api)[0] != 0


def test_hypotheses_have_the_rows_of_stats_M_after_every_call_that_leaves_them(api):
    """Each call draws with its own M, different from the previous call's, and Context.hypotheses() reads them back."""
    import torch
    sc = {m: make_scene(E=2, H=30, W=40, M=m, sub=8, seed=5) for m in (16, 24, 40, 48, 56)}

    def check(m, scores=None):
        assert api.last_stats()["M"] == m
        hy = api.last_hypotheses()
        assert len(hy["scores"]) == m and hy["poses"].shape == (m, 6) and hy["cells"].shape == (m, 4, 2)
        if scores is not None:
            assert np.array_equal(hy["scores"], scores)
        prof = api.context().sample_profile()
        assert prof["lanes"] >= 1

    s = sc[16]
    api.set_seed(1)
    api.forward(s.coords, s.assign, np.zeros((4, 4), np.float32), *s.params)
    check(16)
    s = sc[24]
    api.set_seed(2)
    api.backward(s.coords, np.zeros_like(s.coords), s.assign, s.gt_pose, *W_LOSS, *s.params)
    check(24)
    assert len(api.last_hypotheses(losses=True)["losses"]) == 24
    s = sc[40]
    api.set_seed(3)
    scores, *_ = api.hypotheses_forward(torch.from_numpy(s.coords).cuda(), s.assign, *s.params)
    check(40, scores.cpu().numpy())
    s = sc[48]
    api.set_seed(4)
    api.forward_batch(np.stack([s.coords] * 2), np.stack([s.assign] * 2), np.zeros((2, 4, 4), np.float32), *s.params)
    check(48)
    s = sc[56]
    api.set_seed(5)
    pack = torch.zeros(56 + api.PACK_TAIL, dtype=torch.float64, device="cuda")
    api.forward_pack(torch.from_numpy(s.coords).cuda(), torch.from_numpy(s.assign).cuda(), s.params, 0, pack)
    torch.cuda.synchronize()
    check(56)
    ctx = api.context()
    assert ctx.lib.esacb200_copy_last_scores(ctx.handle, np.zeros(56).ctypes.data, 48) != 0  # M is the last call's


def test_batches_on_worker_contexts_leave_no_hypotheses(api, sc):
    _forward(api, sc)
    api.set_seed(9)
    B = 2
    g = np.zeros((B,) + sc.coords.shape, np.float32)
    api.backward_batch(np.stack([sc.coords] * B), g, np.stack([sc.assign] * B), np.stack([sc.gt_pose] * B), *W_LOSS,
                       *sc.params)
    assert _get_hypotheses(api)[0] != 0
    assert _copy_last_scores(api) is None
