"""The backward's gradient term by term on the GPU (run with `-m gpu`): esac.backward on an odd-sub-sampled, shifted scene, and
the hypotheses node isolated -- api.hypotheses_backward against oracle.esac_oracle.hypotheses_vjp fed the very same upstream
arrays -- with path I alone, path II alone, a random upstream and the DSAC*-style loss of
examples/custom_loss_step_synthetic.py.  Every gradient is compared class by class (tests/grad_terms.py): minimal-set cells,
final inlier cells and the rest, each against its own largest oracle entry.

Measured on an H100 SXM (80 GB, 700 W), worst class of each test (error over the class's own maximum):
  odd-sub-sampled, shifted scene    minimal 8.0e-7, inlier 9.3e-8, rest 2.9e-6
  node, path I alone                0 in every class
  node, path II alone               minimal 6.3e-8, inlier 0, rest 0
  node, random upstream             minimal 1.9e-9, inlier 0, rest 0
  node, DSAC* loss                  minimal 8.8e-9, inlier 0, rest 0
The node's bar of 1e-6 is about 10x its worst class, and leaves a float32 rounding step (<= 1.2e-7 of a cell) where nothing
was measured."""
import runpy
from pathlib import Path

import numpy as np
import pytest

import grad_terms as GT
from esac_b200.synth import make_scene
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

REF_LOSS = (1.0, 100.0, 100.0)   # wLossRot, wLossTrans, lossCut
BAR_ODD = {"minimal": 8e-6, "inlier": 1e-6, "rest": 3e-5}
BAR_NODE = 1e-6
# E = 2, 24x32, M = 32 with 90 % outliers: every hypothesis contributes, 22 carry path I, and both `> 10` clamps trip
# (J_R on six hypotheses, dPNP on two), so the node is checked on each branch of the refinement's derivative
NODE_SCENE, NODE_SEED = dict(E=2, H=24, W=32, M=32, sub=8, seed=31, outlier_frac=0.9), 61


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


def test_backward_terms_on_an_odd_sub_sampled_shifted_scene(api):
    """sub = 5 (pixel centre x*5 + 2), both shifts non-zero and a 27x35 map: six contributing hypotheses."""
    sc = make_scene(E=2, H=27, W=35, M=40, sub=5, seed=23, shiftX=-3, shiftY=4, outlier_frac=0.5)
    g_ref = np.zeros_like(sc.coords)
    l_ref, bt = O.backward(sc.coords, g_ref, sc.assign, sc.gt_pose, *REF_LOSS, *sc.params, seed=73, trace=True)
    api.set_seed(73)
    g = np.zeros_like(sc.coords)
    loss = api.backward(sc.coords, g, sc.assign, sc.gt_pose, *REF_LOSS, *sc.params)
    assert api.last_stats()["n_contrib"] == int((bt.probs >= O.PROB_THRESH).sum()) >= 4
    assert abs(loss - l_ref) < 1e-6 * max(1.0, abs(l_ref))
    rep = GT.assert_classwise(g, g_ref, GT.cell_classes(sc.coords.shape, sc.assign, bt), BAR_ODD, "odd sub")
    print(f"odd sub: {GT.fmt(rep)}")
    assert rep["inlier"]["cells"] > 0 and rep["minimal"]["cells"] > 0


@pytest.fixture(scope="module")
def node(api):
    """The node scene's hypotheses forward on the GPU: (scene, CUDA coordinates, tape, scores, poses, contributing)."""
    import torch
    sc = make_scene(**NODE_SCENE)
    coords = torch.from_numpy(sc.coords).cuda()
    api.set_seed(NODE_SEED)
    scores, poses, contrib, tape = api.hypotheses_forward(coords, sc.assign, *sc.params)
    return sc, coords, tape, scores.cpu().numpy(), poses.cpu().numpy(), contrib.cpu().numpy()


def _reference_upstream(node):
    """p_h dLoss_h and p_h (l_h - E) of the reference loss at the node's refined poses (float64 [M,6], [M])."""
    sc, _, _, scores, poses, _ = node
    gt = sc.gt_pose.astype(np.float64)
    gt_r, gt_t = O.trans2pose(gt)
    p = O.softmax(scores)
    losses = np.array([O.loss(O.pose2trans(q[:3], q[3:]), gt, *REF_LOSS) for q in poses])
    dl = np.array([O.d_loss(q[:3], q[3:], gt_r, gt_t, *REF_LOSS).ravel() for q in poses])
    return p[:, None] * dl, p * (losses - (p * losses).sum())


def _node_against_the_oracle(api, node, grad_poses, grad_scores, what):
    import torch
    sc, coords, tape, _, _, contrib = node
    g = torch.zeros(sc.coords.shape, device="cuda")
    api.hypotheses_backward(tape, coords, g, None if grad_scores is None else torch.tensor(grad_scores, device="cuda"),
                            None if grad_poses is None else torch.tensor(grad_poses, device="cuda"))
    g = g.cpu().numpy()
    g_ref, tr = O.hypotheses_vjp(sc.coords, sc.assign, *sc.params, NODE_SEED, grad_poses, grad_scores)
    assert np.array_equal(contrib, tr.probs >= O.PROB_THRESH)
    assert np.abs(g_ref).max() > 0
    rep = GT.assert_classwise(g, g_ref, GT.cell_classes(sc.coords.shape, sc.assign, tr), BAR_NODE, what)
    print(f"{what}: {GT.fmt(rep)}")
    return rep, tr


def test_node_path_one_alone_meets_the_oracle(api, node):
    """gradScores = None, gradPoses = p dLoss: only the refinement's derivative; the cells outside the inlier sets get nothing."""
    gp, _ = _reference_upstream(node)
    rep, tr = _node_against_the_oracle(api, node, gp, None, "path I")
    assert len(tr.clamped_jr) > 0 and rep["inlier"]["scale"] > 0


def test_node_path_two_alone_meets_the_oracle(api, node):
    """gradPoses = None, gradScores = p (l - E): dScore and the dPNP support at the initial poses."""
    _, gs = _reference_upstream(node)
    rep, tr = _node_against_the_oracle(api, node, None, gs, "path II")
    assert len(tr.clamped_dpnp) > 0 and rep["minimal"]["scale"] > 0


def test_node_random_upstream_meets_the_oracle(api, node):
    sc, *_, contrib = node
    M = sc.assign.shape[0]
    rng = np.random.default_rng(21)
    gp = np.where(contrib[:, None], rng.normal(size=(M, 6)), 0.0)
    gs = np.where(contrib, rng.normal(size=M), 0.0)
    _node_against_the_oracle(api, node, gp, gs, "random upstream")


def test_node_dsac_star_loss_meets_the_oracle(api, node):
    """softmax(scores) . max(angle in degrees, translation error in cm), the loss of examples/custom_loss_step_synthetic.py,
    differentiated in torch (float64) at the node's outputs; its upstream then drives both the node and the oracle."""
    import torch
    from esac_b200.autograd import pose_to_transform
    sc, _, _, scores, poses, _ = node
    ex = Path(__file__).resolve().parents[1] / "examples" / "custom_loss_step_synthetic.py"
    dsac_star_loss = runpy.run_path(str(ex), run_name="example")["dsac_star_loss"]
    s = torch.tensor(scores, requires_grad=True)
    q = torch.tensor(poses, requires_grad=True)
    L = (torch.softmax(s, 0) * dsac_star_loss(pose_to_transform(q), torch.from_numpy(sc.gt_pose).double())).sum()
    gs, gp = (t.numpy() for t in torch.autograd.grad(L, (s, q)))
    assert np.abs(gp).max() > 0 and np.abs(gs).max() > 0
    _node_against_the_oracle(api, node, gp, gs, "DSAC* loss")
