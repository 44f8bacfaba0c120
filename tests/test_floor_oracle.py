"""The oracle's hypotheses node at a probability floor of the caller's (tests/floor_terms.py), on the CPU.

At the default floor it is oracle.esac_oracle.hypotheses_vjp bit for bit.  At floor 0 every hypothesis is refined and
differentiated, and the one term that is an exact derivative, d score / d sceneCoordinates at a fixed pose (the direct
dScore term), matches central differences of a float64 restatement of the score for a loss that weighs every hypothesis,
those far below PROB_THRESH included.  The default floor drops those hypotheses' share."""
import cv2
import numpy as np
import pytest

import floor_terms as FT
from esac_b200.synth import make_scene
from oracle import esac_oracle as O

# 12 of the 16 hypotheses lie below PROB_THRESH, down to p ~ 5e-16
SCENE = dict(E=2, H=8, W=10, M=16, sub=8, seed=3, outlier_frac=0.5)
SEED = 5


@pytest.fixture(scope="module")
def sc():
    return make_scene(**SCENE)


def test_default_floor_is_the_oracle(sc):
    M = sc.assign.shape[0]
    rng = np.random.default_rng(2)
    gp, gs = rng.normal(size=(M, 6)), rng.normal(size=M)
    g, tr = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, gp, gs)
    g_ref, tr_ref = O.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, gp, gs)
    assert np.array_equal(g, g_ref) and np.array_equal(tr.probs, tr_ref.probs)
    assert np.array_equal(tr.gate, tr_ref.probs >= O.PROB_THRESH)
    for h in range(M):
        assert np.array_equal(tr.ref[h][0], tr_ref.ref[h][0]) and np.array_equal(tr.ref[h][1], tr_ref.ref[h][1])


def test_floor_zero_refines_and_differentiates_every_hypothesis(sc):
    M = sc.assign.shape[0]
    gp = np.ones((M, 6))
    _, tr0 = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, gp, None, prob_thresh=0.0)
    _, tr = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, gp, None)
    below = np.nonzero(tr.probs < O.PROB_THRESH)[0]
    assert len(below) >= 8 and tr0.gate.all()
    assert all(tr.grad_I[h] is None for h in below)
    assert sum(tr0.inlier_maps[h] is not None for h in below) >= 4
    assert sum(np.abs(tr0.grad_I[h]).max() > 0 for h in below) >= 4
    # an intermediate floor takes exactly p >= floor
    floor = float(np.sort(tr.probs)[M // 2])
    _, trm = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, gp, None, prob_thresh=floor)
    assert np.array_equal(trm.gate.astype(bool), tr.probs >= floor)
    assert [h for h in range(M) if trm.inlier_maps[h] is not None] == [h for h in range(M) if trm.gate[h] and
                                                                      tr0.inlier_maps[h] is not None]


def _score64(sc, plane, rvec, tvec, samp):
    """getHypScores of one hypothesis in float64: no float rounding of the projection, so it can be differenced."""
    H, W = plane.shape[1:]
    R, _ = cv2.Rodrigues(rvec)
    xc = plane.reshape(3, -1).T.astype(np.float64) @ R.T + tvec.ravel()
    u = xc[:, 0] / xc[:, 2] * sc.f + sc.ppx
    v = xc[:, 1] / xc[:, 2] * sc.f + sc.ppy
    px = samp[:, :, 0].reshape(-1).astype(np.float64)
    py = samp[:, :, 1].reshape(-1).astype(np.float64)
    err = np.minimum(np.sqrt((u - px) ** 2 + (v - py) ** 2), sc.max_reproj)
    return (sc.alpha / (H * W)) * np.sum(1 - 1 / (1 + np.exp(-sc.beta * (err - sc.tau))))


def test_floor_zero_direct_score_gradient_matches_finite_differences(sc):
    """L = sum_h s_h^2 / 2, a loss that is not softmax-weighted and reaches every hypothesis: upstream g_h = s_h.  Per
    hypothesis, the oracle's direct term (grad_II less its dPNP support, which differentiates the minimal-set pose through
    P3P) along a random direction d matches g_h times central differences of the float64 score at the fixed pose."""
    E, _, H, W = sc.coords.shape
    M = sc.assign.shape[0]
    samp = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY)
    _, tr = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, None, None, prob_thresh=0.0)
    gs = np.asarray(tr.scores, np.float64)
    rng = np.random.default_rng(0)
    d = rng.normal(size=sc.coords.shape).astype(np.float32)
    eps = 5e-4
    cp, cm = (sc.coords + eps * d).astype(np.float32), (sc.coords - eps * d).astype(np.float32)
    an = {}
    for floor in (0.0, O.PROB_THRESH):
        _, t = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, SEED, None, gs, prob_thresh=floor)
        row = np.zeros(M)
        for h in range(M):
            direct = t.grad_II[h].copy()
            for i, (x, y) in enumerate(t.hyps[h].cells):
                direct[y * W + x] -= t.support[h][i]
            row[h] = float((direct * d[sc.assign[h]].transpose(1, 2, 0).reshape(H * W, 3)).sum())
        an[floor] = row
    fd = np.array([gs[h] * (_score64(sc, cp[sc.assign[h]], hy.rvec, hy.tvec, samp) -
                            _score64(sc, cm[sc.assign[h]], hy.rvec, hy.tvec, samp)) / (2 * eps)
                   for h, hy in enumerate(tr.hyps)])
    assert np.corrcoef(fd, an[0.0])[0, 1] > 0.995
    assert np.abs(fd - an[0.0]).max() < 0.05 * np.abs(fd).max()
    # the default floor drops the share of the hypotheses below PROB_THRESH, which is not small under this loss
    below = tr.probs < O.PROB_THRESH
    assert not an[O.PROB_THRESH][below].any()
    assert np.abs(fd[below]).max() > 0.2 * np.abs(fd).max()
