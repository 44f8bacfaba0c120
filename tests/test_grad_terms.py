"""The oracle's per-term backward and the class-wise gradient comparator (CPU).

oracle.esac_oracle.hypotheses_vjp is the reference the GPU hypotheses node is held to: under the reference loss's own upstream
it must be backward() bit for bit, and it must be linear in its upstream.  tests/grad_terms.py holds each class of cells
(minimal sets, final inlier sets, the rest) to its own scale: the oracle meets the compiled reference's fixtures that way to
~1e-8, and the comparator must catch errors in path I, in dScore and in the dPNP support that the old bar of 1e-3 of the
largest entry lets through."""
import numpy as np
import pytest

import grad_terms as GT
from esac_b200.synth import make_scene
from oracle import esac_oracle as O
from ref_golden_util import REF_GOLD, params_of

REF_LOSS = (1.0, 100.0, 100.0)
# two scenes of tests/test_gpu_backward.py::test_backward_matches_oracle and its forced scene, with their seeds
SCENES = {
    "s1": (dict(E=1, H=30, W=40, M=32, sub=8, seed=1), 51),
    "s2": (dict(E=3, H=30, W=40, M=48, sub=8, seed=2), 52),
    "forced": (dict(E=3, H=48, W=64, M=48, sub=8, seed=17, outlier_frac=0.9), 57),
}
POWER_BAR = GT.FORCED_BARS   # the bars the GPU tests hold the forced scene to


def _backward(name):
    kw, seed = SCENES[name]
    sc = make_scene(**kw)
    g = np.zeros_like(sc.coords)
    _, bt = O.backward(sc.coords, g, sc.assign, sc.gt_pose, *REF_LOSS, *sc.params, seed=seed, trace=True)
    return sc, seed, g, bt


@pytest.fixture(scope="module")
def forced():
    return _backward("forced")


def _reference_upstream(sc, bt):
    """backward()'s own upstream: p_h dLoss_h at the refined poses, and p_h l_h - sum_j p_h p_j l_j in its order."""
    gt_r, gt_t = O.trans2pose(np.asarray(sc.gt_pose, np.float32).astype(np.float64))
    M = len(bt.probs)
    gp = np.array([bt.probs[h] * O.d_loss(*bt.ref[h], gt_r, gt_t, *REF_LOSS).ravel() for h in range(M)])
    gs = np.zeros(M)
    for h in range(M):
        gs[h] = bt.probs[h] * bt.losses[h]
        for j in range(M):
            gs[h] -= bt.probs[h] * bt.probs[j] * bt.losses[j]
    return gp, gs


@pytest.mark.parametrize("name", list(SCENES))
def test_hypotheses_vjp_under_the_reference_loss_is_backward(name, forced):
    sc, seed, g, bt = forced if name == "forced" else _backward(name)
    gp, gs = _reference_upstream(sc, bt)
    gv, tr = O.hypotheses_vjp(sc.coords, sc.assign, *sc.params, seed, gp, gs)
    assert np.array_equal(tr.probs, bt.probs) and tr.losses is None
    assert np.abs(g).max() > 0
    assert np.array_equal(gv, g)
    # the trace holds every term: reassembling it is the gradient, bit for bit
    again = np.zeros_like(g)
    O.assemble(again, sc.assign, bt.probs, bt.mult, bt.grad_I, bt.grad_II)
    assert np.array_equal(again, g)


def _terms64(sc, tr):
    """sum_h mult_h grad_I[h] + grad_II[h] in float64, [E, H*W, 3]."""
    E, _, H, W = sc.coords.shape
    out = np.zeros((E, H * W, 3))
    for h in np.nonzero(tr.probs >= O.PROB_THRESH)[0]:
        out[sc.assign[h]] += tr.mult[h] * tr.grad_I[h] + tr.grad_II[h]
    return out


def test_hypotheses_vjp_is_linear_in_its_upstream():
    kw, seed = SCENES["s2"]
    sc = make_scene(**kw)
    M = sc.assign.shape[0]
    rng = np.random.default_rng(5)
    a1, a2 = rng.normal(size=(M, 6)), rng.normal(size=(M, 6))
    b1, b2 = rng.normal(size=M), rng.normal(size=M)
    t1, t2, t12 = (_terms64(sc, O.hypotheses_vjp(sc.coords, sc.assign, *sc.params, seed, a, b)[1])
                   for a, b in ((a1, b1), (a2, b2), (a1 + a2, b1 + b2)))
    scale = np.abs(t12).max()
    assert scale > 0
    assert np.abs(t12 - (t1 + t2)).max() <= 1e-12 * scale
    # None is zero, and each upstream feeds only its own path
    g0, _ = O.hypotheses_vjp(sc.coords, sc.assign, *sc.params, seed, None, None)
    assert not g0.any()
    _, tr = O.hypotheses_vjp(sc.coords, sc.assign, *sc.params, seed, a1, None)
    assert all(not gi.any() for gi in tr.grad_II) and any(gi is not None and gi.any() for gi in tr.grad_I)


def _small_fixtures():
    return [p for p in REF_GOLD if "coords" in np.load(p).files]


@pytest.mark.parametrize("path", _small_fixtures(), ids=lambda p: p.stem)
def test_oracle_meets_the_compiled_reference_class_by_class(path):
    """Observed: <= 1.1e-8 of each class's own maximum on every small fixture."""
    z = np.load(path)
    g = np.zeros_like(z["coords"])
    w_rot, w_trans, cut = (float(v) for v in z["loss_args"])
    _, bt = O.backward(z["coords"], g, z["assign"], z["gt_pose"], w_rot, w_trans, cut, *params_of(z),
                       mt=O.ThreadRandStream(1305), trace=True)
    rep = GT.assert_classwise(g, z["grads"], GT.cell_classes(g.shape, z["assign"], bt), 1e-7, path.stem)
    assert rep["minimal"]["cells"] > 0


def _assembled(sc, bt, grad_I=None, grad_II=None):
    g = np.zeros_like(sc.coords)
    O.assemble(g, sc.assign, bt.probs, bt.mult, bt.grad_I if grad_I is None else grad_I,
               bt.grad_II if grad_II is None else grad_II)
    return g


def _without_support(sc, bt, h, grad_II):
    """grad_II[h] less its dPNP support (the support sits on the hypothesis's minimal-set cells)."""
    W = sc.coords.shape[3]
    out = grad_II.copy()
    for i, (x, y) in enumerate(bt.hyps[h].cells):
        out[y * W + x] -= bt.support[h][i]
    return out


def test_the_comparator_catches_what_the_global_bar_lets_through(forced):
    """Each perturbation of one term of the forced scene's oracle gradient fails the class-wise check at the bar the GPU tests
    use; the first two pass the old bar of 1e-3 of the largest entry, which is the gap the class-wise check closes."""
    sc, _, g, bt = forced
    classes = GT.cell_classes(sc.coords.shape, sc.assign, bt)
    assert np.array_equal(_assembled(sc, bt), g)
    assert not GT.failures(GT.compare(g, g, classes), POWER_BAR)
    contrib = np.nonzero(bt.probs >= O.PROB_THRESH)[0]
    size_I = {h: np.abs(bt.probs[h] * bt.grad_I[h]).max() for h in contrib}
    carrying = [h for h in contrib if size_I[h] > 0]
    assert len(carrying) >= 8

    def fails(g_bad):
        return GT.failures(GT.compare(g_bad, g, classes), POWER_BAR)

    # 1. drop the path I of the hypothesis whose path I is the smallest
    h = min(carrying, key=size_I.get)
    grad_I = list(bt.grad_I)
    grad_I[h] = np.zeros_like(grad_I[h])
    bad = fails(_assembled(sc, bt, grad_I=grad_I))
    assert bad == ["inlier"], (h, bad)
    # 2. path I of every hypothesis 0.1 % too large
    bad = fails(_assembled(sc, bt, grad_I=[None if gi is None else gi * (1 + 1e-3) for gi in bt.grad_I]))
    assert "inlier" in bad and "global" not in bad, bad
    # 3. the direct dScore term of one expert's hypotheses with the wrong sign
    e = int(sc.assign[contrib[0]])
    grad_II = list(bt.grad_II)
    for k in contrib:
        if sc.assign[k] == e:
            direct = _without_support(sc, bt, k, bt.grad_II[k])
            grad_II[k] = bt.grad_II[k] - 2 * direct
    bad = fails(_assembled(sc, bt, grad_II=grad_II))
    assert "rest" in bad, bad
    # 4. the dPNP support of the hypothesis whose support is the smallest non-zero one
    size_S = {k: np.abs(bt.support[k]).max() for k in contrib if np.abs(bt.support[k]).max() > 0}
    h = min(size_S, key=size_S.get)
    grad_II = list(bt.grad_II)
    grad_II[h] = _without_support(sc, bt, h, bt.grad_II[h])
    bad = fails(_assembled(sc, bt, grad_II=grad_II))
    assert "minimal" in bad, (h, bad)
