"""The device at every camera orientation, not only within 30 degrees of the world axes (run with `-m gpu`).

a. The pose loss on the device (pose_loss_kernel: pose2trans, gt_trans2pose, pose_loss, pose_dloss) on the edge grid of
   tests/pose_loss_grid.py around every orientation of tests/orientations.py, held to the 40-digit yardstick and, at the
   degenerate entries, to the outcome classes of the reference's own dLoss (tests/golden/pin/ref_pose_loss_edges.npz).
b. forward, backward and the hypotheses node on small rotated scenes against the cv2 oracle, with the bars of
   tests/test_gpu_forward.py, tests/test_gpu_backward.py and tests/test_gpu_hypotheses.py.  On the half turn about x every
   good hypothesis sits within noise of the rvec's sign flip, where the central differences of dPNP jump and the > 10
   clamp zeroes a hypothesis's minimal-set term: the device must clamp the same hypotheses as the oracle.
"""
from pathlib import Path

import numpy as np
import pytest

import grad_terms as GT
import pose_loss_grid as G
from esac_b200.synth import make_scene, pose_error
from oracle import esac_oracle as O
from orientations import NAMES, ORIENTATIONS

pytestmark = pytest.mark.gpu

PIN = Path(__file__).resolve().parent / "golden" / "pin" / "ref_pose_loss_edges.npz"
SCORE_TOL = 1e-4
ROT_TOL_DEG = 1e-3
TRANS_TOL_M = 1e-5
BAR_SCENES = {"minimal": 2.5e-5, "inlier": 7e-6, "rest": 7.5e-5}   # test_gpu_backward.py's class-wise bars


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


@pytest.fixture(scope="module")
def pin():
    return np.load(PIN)


def test_device_pose_loss_at_every_orientation(api, pin):
    import torch
    worst = {}
    for name in NAMES:
        gt = torch.from_numpy(G.ground_truth(name)).cuda()
        poses = pin[f"{name}_poses"]
        cuts = pin[f"{name}_cuts"]
        losses, dloss = np.zeros(len(poses)), np.zeros((len(poses), 6))
        for cut in np.unique(cuts):
            rows = np.flatnonzero(cuts == cut)
            lo, dl = api.pose_loss(torch.from_numpy(poses[rows]).cuda(), gt, G.W_ROT, G.W_TRANS, float(cut))
            losses[rows], dloss[rows] = lo.cpu().numpy(), dl.cpu().numpy()
        worst[name] = G.check_pose_loss(name, losses, dloss, pin)
    print("worst error / bar (loss, dloss):", {k: tuple(round(float(x), 3) for x in v) for k, v in worst.items()})


# ---- end to end --------------------------------------------------------------------------------------------------------
# E = 2, 30x40, M = 32; the seeds keep the two best scores more than 0.3 apart
SCENES = [("pi_x", 1), ("pi_n", 1), ("179.99_n", 1), ("90_n", 2), ("uniform0", 1), ("uniform3", 2)]


def _scene(name, seed):
    return make_scene(E=2, H=30, W=40, M=32, sub=8, seed=seed, rotation=ORIENTATIONS[name])


def _rot_deg(Ra, Rb):
    Ta = np.eye(4); Ta[:3, :3] = Ra
    Tb = np.eye(4); Tb[:3, :3] = Rb
    return pose_error(Ta, Tb)[0]


def _same_hypotheses(hy, hyps):
    """The same tries and cells, and the same sampled poses compared as rotations (r and -r agree at pi)."""
    assert np.array_equal(hy["tries"], np.array([h.tries for h in hyps]))
    assert np.array_equal(hy["cells"], np.array([[list(c) for c in h.cells] for h in hyps]))
    for p, h in zip(hy["poses"], hyps):
        Ta = O.pose2trans(p[:3], p[3:])
        Tb = O.pose2trans(h.rvec, h.tvec)
        rot, trans = pose_error(Ta, Tb)
        assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (rot, trans)


@pytest.mark.parametrize("name,seed", SCENES, ids=[s[0] for s in SCENES])
def test_forward_matches_oracle_at_any_orientation(api, name, seed):
    sc = _scene(name, seed)
    ref_pose = np.zeros((4, 4), np.float32)
    ref_e, tr = O.forward(sc.coords, sc.assign, ref_pose, *sc.params, seed=60 + seed, trace=True)
    api.set_seed(60 + seed)
    out = np.zeros((4, 4), np.float32)
    e = api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    st = api.last_stats()
    _same_hypotheses(hy, tr.hyps)
    assert np.abs(hy["scores"] - np.array(tr.scores)).max() < SCORE_TOL
    s = np.sort(np.array(tr.scores))[::-1]
    assert s[0] - s[1] > 10 * SCORE_TOL
    assert st["winner"] == tr.winner and e == ref_e
    assert st["refine_rounds"] == tr.rounds
    rot, trans = pose_error(out, ref_pose)
    assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (rot, trans)
    ref6 = hy["refined"][tr.winner]
    rot, trans = pose_error(O.pose2trans(ref6[:3].reshape(3, 1), ref6[3:].reshape(3, 1)), O.pose2trans(tr.ref_rvec, tr.ref_tvec))
    assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (rot, trans)
    # the estimate is the rotated camera
    assert _rot_deg(out[:3, :3].astype(np.float64), sc.gt_pose[:3, :3].astype(np.float64)) < 5.0


@pytest.mark.parametrize("name,seed", SCENES, ids=[s[0] for s in SCENES])
def test_backward_matches_oracle_at_any_orientation(api, name, seed):
    sc = _scene(name, seed)
    g_ref = np.zeros_like(sc.coords)
    l_ref, bt = O.backward(sc.coords, g_ref, sc.assign, sc.gt_pose, 1.0, 100.0, 100.0, *sc.params, seed=60 + seed, trace=True)
    if name == "pi_x":
        assert len(bt.clamped_dpnp) > 0   # the rvec-flip edge of dPNP's central differences is exercised
    api.set_seed(60 + seed)
    g = np.zeros_like(sc.coords)
    loss = api.backward(sc.coords, g, sc.assign, sc.gt_pose, 1.0, 100.0, 100.0, *sc.params)
    hy = api.last_hypotheses(losses=True)
    st = api.last_stats()
    _same_hypotheses(hy, bt.hyps)
    assert np.abs(hy["scores"] - np.array(bt.scores)).max() < SCORE_TOL
    assert st["n_contrib"] == int((bt.probs >= O.PROB_THRESH).sum())
    assert np.abs(hy["losses"] - np.array(bt.losses)).max() < 1e-5 * max(1.0, np.abs(bt.losses).max())
    assert abs(loss - l_ref) < 1e-6 * max(1.0, abs(l_ref))
    rep = GT.assert_classwise(g, g_ref, GT.cell_classes(sc.coords.shape, sc.assign, bt), BAR_SCENES, name)
    print(f"{name}: {GT.fmt(rep)}")


@pytest.mark.parametrize("name,seed", SCENES, ids=[s[0] for s in SCENES])
def test_reference_loss_through_the_node_meets_the_oracle_at_any_orientation(api, name, seed):
    import torch
    from esac_b200.autograd import esac_hypotheses, reference_pose_loss
    sc = _scene(name, seed)
    g_ref = np.zeros_like(sc.coords)
    l_ref, bt = O.backward(sc.coords, g_ref, sc.assign, sc.gt_pose, 1.0, 100.0, 100.0, *sc.params, seed=60 + seed, trace=True)
    coords = torch.from_numpy(sc.coords).cuda().requires_grad_(True)
    api.set_seed(60 + seed)
    scores, poses, _ = esac_hypotheses(coords, torch.from_numpy(sc.assign).cuda(), *sc.params)
    losses = reference_pose_loss(poses, torch.from_numpy(sc.gt_pose).cuda(), 1.0, 100.0, 100.0)
    L = (torch.softmax(scores, 0) * losses).sum()
    L.backward()
    assert np.abs(scores.detach().cpu().numpy() - np.array(bt.scores)).max() < SCORE_TOL
    assert abs(L.item() - l_ref) < 1e-6 * max(1.0, abs(l_ref))
    g = coords.grad.cpu().numpy()
    rep = GT.assert_classwise(g, g_ref, GT.cell_classes(sc.coords.shape, sc.assign, bt), BAR_SCENES, name)
    print(f"{name}: {GT.fmt(rep)}")
