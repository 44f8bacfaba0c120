"""The pose pipeline against the oracle away from the reference's default hyperparameters (run with `-m gpu` on an H100).

Every other parity test runs at tau = 10 px, beta = 0.5, maxReproj = 100, alpha = 100 and the loss (1, 100, 100), but the
kernels branch on these values: the prefilter's band max(2 tau, 4 px) and its window-cut hint at sample_hint * tau, the
exact verdict's early exit at 1.25 tau + 1 px, the scoring kernel's fold (k1 = beta log2 e >= 1e-3 and tmax <= 63), the
refinement pretest's band around tau and its guard tau <= maxReproj, and the stream-ordered backward, which reads sub, tau,
alpha, beta and maxReproj from the tape header.  Each check below uses the oracle and the bars of its default-parameter
twin: test_gpu_sample_schedules.py (tries and cells exactly, poses to 1e-8), test_gpu_score_shapes.py (1e-4 at alpha 100),
test_gpu_forward.py (rounds and inliers exactly, poses to 1e-3 deg / 1e-5 m), test_gpu_backward.py (class-wise bars),
test_gpu_hypotheses.py and the stream-ordered tests (bitwise)."""
import dataclasses
import itertools

import numpy as np
import pytest

import grad_terms as GT
import minimal_sets as MS
from esac_b200.synth import make_scene, pose_error
from oracle import esac_oracle as O
from oracle import score_fp64
from test_gpu_forward import ROT_TOL_DEG, TRANS_TOL_M, perturbed_truth
from test_gpu_sample_schedules import _assert_matches, _oracle, _restore, _sample
from test_gpu_score_shapes import _dense_poses, score_forced
from test_host_thresholds import counterexample

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-4                                   # at alpha = 100; scores scale with alpha, so does the bar
BAR_SCENES = {"minimal": 2.5e-5, "inlier": 7e-6, "rest": 7.5e-5}   # test_gpu_backward.py's class-wise bars
LOG2E = 1.4426950408889634


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


@pytest.fixture(autouse=True)
def library_defaults(api):
    try:
        yield
    finally:
        _restore(api)


def with_params(sc, **kw):
    return dataclasses.replace(sc, **kw)


# ---- sampling ----------------------------------------------------------------------------------------------------------
SAMPLE_TAUS = (0.5, 1.0, 2.0, 25.0, 100.0)
SAMPLE_SEED = 611


def sample_scene(tau):
    """Low noise and every hypothesis on the true expert, so each ends in a few tries even at sub-pixel tau (a wrong expert
    there can need up to 1e6)."""
    sc = make_scene(E=2, H=30, W=40, M=48, sub=8, seed=61, noise=5e-4, outlier_frac=0.2, shiftX=2, shiftY=-3)
    sc = with_params(sc, tau=tau)
    sc.assign[:] = sc.gt_expert
    return sc


@pytest.fixture(scope="module")
def sampled():
    return {tau: (sample_scene(tau), _oracle(sample_scene(tau), SAMPLE_SEED)) for tau in SAMPLE_TAUS}


@pytest.mark.parametrize("hint", [None, 0.0], ids=["hint_default", "hint_off"])
@pytest.mark.parametrize("tau", SAMPLE_TAUS)
def test_sampling_matches_oracle_at_tau(api, sampled, tau, hint):
    sc, ref = sampled[tau]
    opts = {} if hint is None else dict(sample_hint=hint)
    hy, prof, _, _ = _sample(api, sc, SAMPLE_SEED, **opts)
    print(tau, hint, prof, "tries max", ref.tries.max())
    _assert_matches(hy, ref)
    assert ref.tries.max() > 1                       # not every first try passed
    assert ref.tries.max() < O.MAX_SAMPLING_TRIES


@pytest.mark.parametrize("hint", [None, 0.0], ids=["hint_default", "hint_off"])
def test_subpixel_counterexample_is_accepted_on_its_first_try(api, hint):
    """A minimal set the exact path accepts at tau = 0.5 (4th point 0.4537 px off under its P3P pose), whose float 4th
    point on the host compile lies outside a band of 2 tau (tests/test_host_thresholds.py): injected as the first candidate
    of every hypothesis, the device must stop at try 1, as the oracle does."""
    sc, _, _, cells = counterexample()
    sc = with_params(sc, tau=0.5)
    M = 6
    sc.assign = np.full(M, sc.gt_expert, np.int64)
    inject = np.repeat(np.asarray(cells, np.int32)[None, None], 2, axis=1).repeat(M, axis=0)   # [M, 2, 4, 2]
    ref = _oracle(sc, 0, 2, inject)
    assert ref.tries.tolist() == [1] * M
    opts = {} if hint is None else dict(sample_hint=hint)
    hy, _, _, _ = _sample(api, sc, 0, inject=inject, **opts)
    assert hy["tries"].tolist() == [1] * M, hy["tries"]
    _assert_matches(hy, ref)


# ---- the device's verdicts at sub-pixel tau ----------------------------------------------------------------------------
# The device compile of the prefilter (MUFU approximations, contracted FMAs) has its own float error, so the band's floor is
# held on the device too: true-expert tries that the exact path accepts (and some it rejects) are drawn on the host, injected
# as the first try of a hypothesis each, and every device verdict must equal the cv2 oracle's.  Maps of 640 x 480 px images
# (principal point 320, 240), as minimal_sets.root_errors assumes when it arbitrates a rounding tie.
SWEEP_TAUS = (0.05, 0.1, 0.2, 0.3, 0.5, 0.75, 1.0)
SWEEP_SCENES = {
    "room-noise2e-3": dict(E=2, H=60, W=80, M=8, sub=8, seed=2, noise=0.002, active_only=False),    # the host counterexample's
    "room-noise5e-4": dict(E=2, H=60, W=80, M=8, sub=8, seed=3, noise=5e-4, active_only=False),
    "room-noise1e-2-shift": dict(E=2, H=60, W=80, M=8, sub=8, seed=4, noise=0.01, shiftX=3, shiftY=-5, active_only=False),
    "outdoor-world700": dict(E=2, H=60, W=80, M=8, sub=8, seed=5, noise=0.01, outdoor=True, world_offset=700.0,
                             active_only=False),
    "room-millimetres": dict(E=2, H=60, W=80, M=8, sub=8, seed=6, noise=0.002, unit_scale=1000.0, active_only=False),
    "room-sub4": dict(E=2, H=120, W=160, M=8, sub=4, seed=7, noise=0.005, active_only=False),
}
SWEEP_DRAWS = 40000        # true-expert draws per scene
SWEEP_ACC, SWEEP_REJ = 3000, 600   # per scene and tau: accepted tries, and tries the prefilter passes but the exact path rejects


def sweep_tries(lib, sc, obj, img, tau):
    """Indices of the draws injected at tau: up to SWEEP_ACC accepted ones and SWEEP_REJ that reach the exact path only to
    be rejected there (host compile)."""
    from test_host_thresholds import tries
    mp, _, ac = tries(lib, obj, img, sc.f, sc.ppx, sc.ppy, tau)
    return np.concatenate([np.flatnonzero(ac)[:SWEEP_ACC], np.flatnonzero(mp & ~ac)[:SWEEP_REJ]])


def sweep_draws(name):
    from test_host_thresholds import draws
    sc = make_scene(**SWEEP_SCENES[name])
    obj, img = draws(sc, sc.gt_expert, SWEEP_DRAWS, np.random.default_rng(500 + list(SWEEP_SCENES).index(name)))
    cells = (img + np.array([sc.shiftX, sc.shiftY]) - sc.sub // 2) // sc.sub
    return sc, obj, img, cells.astype(np.int32)


def _disagreements(lib, dev_acc, ref_acc, objs, imgs, f, tau):
    """Hypotheses whose device verdict differs from the oracle's, less rounding ties shown at 40 digits."""
    out = []
    for h in np.flatnonzero(dev_acc != ref_acc):
        if not MS.rounding_tie(MS.root_errors(lib, objs[h], imgs[h], f), tau=tau):
            out.append(int(h))
    return out


@pytest.mark.parametrize("tau", SWEEP_TAUS)
def test_device_verdicts_on_random_draws_at_subpixel_tau(api, tau):
    lib = api.load_library()
    n_acc = n_all = 0
    dropped = []
    for name in SWEEP_SCENES:
        sc, obj, img, cells = sweep_draws(name)
        sc = with_params(sc, tau=tau)
        sel = sweep_tries(lib, sc, obj, img, tau)
        sc.assign = np.full(len(sel), sc.gt_expert, np.int64)
        inject = np.repeat(cells[sel][:, None], 2, axis=1)                # [M, 2, 4, 2]: the try, then itself again
        ref = _oracle(sc, 0, 2, inject)
        hy, _, _, _ = _sample(api, sc, 0, inject=inject)
        dev_acc, ref_acc = hy["tries"] == 1, ref.tries == 1
        bad = _disagreements(lib, dev_acc, ref_acc, obj[sel], img[sel].astype(np.float32), sc.f, tau)
        dropped += [(name, int(sel[h]), bool(dev_acc[h])) for h in bad]
        n_acc += int(ref_acc.sum())
        n_all += len(sel)
    print(f"tau {tau:g}: {n_all} injected tries, {n_acc} accepted by the oracle, {len(dropped)} device verdicts differ")
    assert not dropped, ("(scene, draw, device accepted) where the device's verdict differs", dropped[:16])
    assert n_acc >= 200                               # 280 at tau = 0.05, over 1e4 from 0.75 up


@pytest.mark.parametrize("tau", SWEEP_TAUS)
def test_device_verdicts_on_crafted_sets_at_subpixel_tau(api, tau):
    """tests/minimal_sets.py's families with their 4th point over [0, 1.2 tau) of the true pose, scaled and offset, each
    injected as [crafted, anchor] (tests/test_gpu_minimal_sets.py's layout)."""
    lib = api.load_library()
    ts = []
    for fam in MS.FAMILIES:
        base = MS.generate(fam, 80, seed=13, tau=tau)
        ts += base + MS.variants(base)
    pk = MS.pack(ts, 64, 525.0)
    K = O.cam_mat(525.0, MS.PPX, MS.PPY)
    ref = O.sample_hypotheses(pk.coords, pk.assign, O.create_sampling(MS.W, MS.H, MS.SUB, 0, 0), K, 10 ** 6, tau,
                              injected_cells=pk.cells)
    ctx = api.context()
    ctx.set_option("fixed_seed", 1)
    api.set_seed(5)
    api.inject_cells(pk.cells)
    out = np.zeros((4, 4), np.float32)
    api.forward(pk.coords, pk.assign, out, 0, 0, 525.0, MS.PPX, MS.PPY, tau, 100.0, 0.5, 100.0, MS.SUB)
    hy = api.last_hypotheses()
    dev_acc, ref_acc = hy["tries"] == 1, np.array([h.tries == 1 for h in ref])
    bad = _disagreements(lib, dev_acc, ref_acc, [t.obj for t in pk.tries], [t.img() for t in pk.tries], 525.0, tau)
    print(f"tau {tau:g}: {len(pk.tries)} crafted tries, {int(ref_acc.sum())} accepted by the oracle, {len(bad)} differ")
    assert not bad, [(pk.tries[h].params, bool(dev_acc[h])) for h in bad[:8]]
    assert ref_acc.sum() > 0 and np.all(hy["tries"] <= 2)


# true-expert draws of the sweep that the device compile dropped with the parent's band of 2 tau alone (found by the sweep
# above on an H100); the first also with a floor of 1 px
DEVICE_DROPPED = [("room-noise5e-4", 18558, 0.5), ("room-noise5e-4", 12451, 0.2), ("room-noise5e-4", 33404, 0.2)]


@pytest.mark.parametrize("name,draw,tau", DEVICE_DROPPED, ids=[f"{n}-{d}-tau{t:g}" for n, d, t in DEVICE_DROPPED])
def test_device_dropped_tries_are_accepted_on_their_first_try(api, name, draw, tau):
    sc, obj, img, cells = sweep_draws(name)
    sc = with_params(sc, tau=tau)
    M = 6
    sc.assign = np.full(M, sc.gt_expert, np.int64)
    inject = np.repeat(cells[draw][None, None], 2, axis=1).repeat(M, axis=0)         # [M, 2, 4, 2]
    ref = _oracle(sc, 0, 2, inject)
    assert ref.tries.tolist() == [1] * M
    for hint in (None, 0.0):
        hy, _, _, _ = _sample(api, sc, 0, inject=inject, **({} if hint is None else dict(sample_hint=hint)))
        assert hy["tries"].tolist() == [1] * M, (hint, hy["tries"])
        _assert_matches(hy, ref)


# ---- scoring -----------------------------------------------------------------------------------------------------------
# (tau, beta, alpha, maxReproj): tmax = beta log2(e) (maxReproj - tau) - 32 on each side of 63 and far above it, k1 on each
# side of 1e-3, maxReproj below and at tau, alpha 1 and 1000
SCORE_GRID = {
    "tmax61.8": (10.0, 0.5, 100.0, 140.0),
    "tmax65.4": (10.0, 0.5, 100.0, 145.0),
    "maxr1e4": (10.0, 0.5, 100.0, 1e4),
    "k1_above": (10.0, 7.0e-4, 100.0, 100.0),
    "k1_below": (10.0, 6.9e-4, 100.0, 100.0),
    "maxr_below_tau": (40.0, 0.1, 400.0, 30.0),
    "maxr_eq_tau": (25.0, 0.5, 100.0, 25.0),
    "alpha1": (2.0, 2.0, 1.0, 100.0),
    "alpha1000": (0.5, 1.0, 1000.0, 60.0),
    "tau200": (200.0, 0.05, 100.0, 300.0),
}


def folds(tau, beta, max_reproj):
    """score_constants (score.cu) in float32: whether the kernel folds k1 into the pose rows."""
    k1 = np.float32(beta) * np.float32(LOG2E)
    k0s = -np.float32(beta) * np.float32(tau) * np.float32(LOG2E) - np.float32(32)
    tmax = np.float32(max_reproj) * k1 + k0s
    return bool(k1 >= np.float32(1e-3) and tmax <= 63)


def test_score_grid_covers_both_sides_of_the_fold():
    expect = {"tmax61.8": True, "tmax65.4": False, "maxr1e4": False, "k1_above": True, "k1_below": False}
    for name, want in expect.items():
        assert folds(*[SCORE_GRID[name][i] for i in (0, 1, 3)]) == want, name


@pytest.mark.parametrize("name", list(SCORE_GRID))
@pytest.mark.parametrize("H,W,sub", [(120, 160, 4), (61, 81, 3)])
def test_scores_match_fp64_on_the_parameter_grid(api, name, H, W, sub):
    import torch
    tau, beta, alpha, max_reproj = SCORE_GRID[name]
    sc = make_scene(E=3, H=H, W=W, M=36, sub=sub, seed=43, shiftX=3, shiftY=-5, noise=0.01)
    poses = _dense_poses(sc, np.random.default_rng(43), len(sc.assign))
    params = dataclasses.replace(sc, tau=tau, alpha=alpha, beta=beta, max_reproj=max_reproj).params
    ref, _ = score_fp64.score(sc.coords, sc.assign, poses, *params)
    t = torch.from_numpy(sc.coords).cuda()
    a = torch.from_numpy(sc.assign).cuda()
    tol = SCORE_TOL * alpha / 100.0
    for ppt in (2, 8):
        got = score_forced(api, t, a, poses, params, ppt, 16)
        assert np.abs(got - ref).max() < tol, (name, ppt, folds(tau, beta, max_reproj), np.abs(got - ref).max())
    got = api.score_poses(sc.coords, sc.assign, poses, *params)
    assert np.abs(got - ref).max() < tol
    assert ref.max() - ref.min() > 100 * tol                  # the scores tell poses apart


@pytest.mark.parametrize("max_reproj", [140.0, 145.0, 1e4])
def test_single_cell_probes_on_both_sides_of_the_fold(api, max_reproj):
    """test_gpu_score_shapes.py's probe maps (one cell per plane within 3 px of tau, alpha = N, so a score is one probe's
    weight) with maxReproj on each side of the fold's tmax <= 63 and far above it: the probe maps' bar of 1e-5."""
    import torch
    from test_gpu_score_shapes import probe_scene
    coords, assign, poses, params = probe_scene(60, 80, 8, 3, -5, seed=7)
    params = params[:8] + (max_reproj,) + params[9:]
    ref, _ = score_fp64.score(coords, assign, poses, *params)
    assert 0.01 < ref.min() and ref.max() < 0.99
    t = torch.from_numpy(coords).cuda()
    a = torch.from_numpy(assign).cuda()
    for ppt in (2, 8):
        got = score_forced(api, t, a, poses, params, ppt, 5)
        assert np.abs(got - ref).max() < 1e-5, (max_reproj, ppt, np.abs(got - ref).max())


# ---- refinement --------------------------------------------------------------------------------------------------------
REFINE_CASES = {                # name: (tau, maxReproj)
    "tau0.5": (0.5, 100.0),
    "tau2": (2.0, 100.0),
    "tau25": (25.0, 100.0),
    "tau100=maxr": (100.0, 100.0),
    "tau40>maxr30": (40.0, 30.0),
}


@pytest.fixture(scope="module", params=list(REFINE_CASES))
def refine_case(request):
    tau, max_reproj = REFINE_CASES[request.param]
    # above maxReproj every cell is fitted, outliers too: keep them few (each still lies beyond tau unclamped), so that the
    # fit stays well-conditioned
    sc = make_scene(E=2, H=60, W=80, M=12, sub=8, seed=66, noise=0.003, outlier_frac=0.02 if tau > max_reproj else 0.3)
    sc = with_params(sc, tau=tau, max_reproj=max_reproj)
    M = 12
    assign = np.full(M, sc.gt_expert, np.int64)
    # ground truth moved by about tau / 4 px at most, so that sub-pixel thresholds still find inliers to refine on
    poses6 = perturbed_truth(sc, np.random.default_rng(66), M, rot=min(0.002, 0.0005 * tau), trans=min(0.01, 0.0025 * tau))
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    H, W = sc.coords.shape[2:]
    sampling = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY)
    ref = []
    for h in range(M):
        rv, tv = poses6[h, :3].reshape(3, 1), poses6[h, 3:].reshape(3, 1)
        errs, _ = O.get_repro_errs(sc.coords, rv, tv, sc.gt_expert, sampling, K, sc.max_reproj)
        r, t, im, rr = O.refine_hyp(sc.coords, errs, sampling, K, sc.gt_expert, sc.tau, O.MAX_REF_STEPS, sc.max_reproj, rv, tv)
        ref.append((r, t, 0 if im is None else int(im.sum()), rr))
    return request.param, sc, assign, poses6, ref


def test_refinement_matches_oracle_at_tau(api, refine_case):
    """refine_group in {1, auto, max} x refine_compact in {0, 1}: rounds and inlier counts exact, poses within 1e-3 deg /
    1e-5 m of the oracle's refineHyp.  Above maxReproj every clamped error is below tau, so every cell is an inlier and the
    float pretest (which classifies by the unclamped error) must stay off."""
    name, sc, assign, poses6, ref = refine_case
    N = sc.coords.shape[2] * sc.coords.shape[3]
    ctx = api.context()
    try:
        for grp, compact in itertools.product((1, 0, 1 << 20), (0, 1)):
            ctx.set_option("refine_group", grp)
            ctx.set_option("refine_compact", compact)
            got, rounds, inl = api.refine_poses(sc.coords, assign, poses6, sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy, sc.tau,
                                                sc.max_reproj, sc.sub)
            tag = (name, grp, api.last_stats()["refine_group"], compact)
            for h, (r, t, n_in, rr) in enumerate(ref):
                assert rounds[h] == rr and inl[h] == n_in, (tag, h, rounds[h], rr, inl[h], n_in)
                Ta, Tb = O.pose2trans(r, t), O.pose2trans(got[h, :3].reshape(3, 1), got[h, 3:].reshape(3, 1))
                rot, trans = pose_error(Tb, Ta)
                assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (tag, h, rot, trans)
    finally:
        ctx.set_option("refine_group", 0)
        ctx.set_option("refine_compact", 1)
    assert max(r[3] for r in ref) >= 1 and min(r[2] for r in ref) >= 4   # every job was refined
    if sc.tau > sc.max_reproj:                        # every cell is an inlier, also those beyond tau before the clamp
        assert all(r[2] == N for r in ref)
        K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
        sampling = O.create_sampling(sc.coords.shape[3], sc.coords.shape[2], sc.sub, sc.shiftX, sc.shiftY)
        raw, _ = O.get_repro_errs(sc.coords, poses6[0, :3].reshape(3, 1), poses6[0, 3:].reshape(3, 1), sc.gt_expert, sampling,
                                  K, 1e30)
        assert (np.asarray(raw) > sc.tau).sum() >= 20


# ---- backward ----------------------------------------------------------------------------------------------------------
# name: (make_scene arguments, (tau, alpha, beta, maxReproj), (wRot, wTrans, lossCut), seed)
BACKWARD_SETS = {
    "tight_cut": (dict(E=2, H=30, W=40, M=24, sub=8, seed=71, noise=0.005), (4.0, 30.0, 1.0, 60.0), (1.0, 100.0, 0.05), 81),
    "clamp_wrot0": (dict(E=2, H=24, W=32, M=24, sub=8, seed=72), (25.0, 400.0, 0.1, 30.0), (0.0, 100.0, 100.0), 82),
    "above_maxr_wtrans0": (dict(E=2, H=24, W=32, M=24, sub=8, seed=73, outlier_frac=0.02), (40.0, 200.0, 0.2, 30.0), (1.0, 0.0, 100.0), 83),
    "unfolded_alpha1000": (dict(E=2, H=30, W=40, M=24, sub=8, seed=74, noise=0.005), (6.0, 1000.0, 2.0, 100.0),
                           (0.5, 30.0, 5.0), 84),
}


def backward_scene(name):
    kw, (tau, alpha, beta, max_reproj), loss, seed = BACKWARD_SETS[name]
    return with_params(make_scene(**kw), tau=tau, alpha=alpha, beta=beta, max_reproj=max_reproj), loss, seed


@pytest.mark.parametrize("name", list(BACKWARD_SETS))
def test_backward_matches_oracle_away_from_the_defaults(api, name):
    sc, loss_args, seed = backward_scene(name)
    g_ref = np.zeros_like(sc.coords)
    l_ref, bt = O.backward(sc.coords, g_ref, sc.assign, sc.gt_pose, *loss_args, *sc.params, seed=seed, trace=True)
    # the forward's winner and scores first
    out = np.zeros((4, 4), np.float32)
    ref_out = np.zeros((4, 4), np.float32)
    e_ref, tr = O.forward(sc.coords, sc.assign, ref_out, *sc.params, seed=seed, trace=True)
    api.set_seed(seed)
    e = api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    tol = SCORE_TOL * sc.alpha / 100.0
    assert np.abs(hy["scores"] - np.array(tr.scores)).max() < tol
    assert e == e_ref and api.last_stats()["winner"] == tr.winner
    rot, trans = pose_error(out, ref_out)
    assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (rot, trans)
    # then the backward, class by class
    api.set_seed(seed)
    g = np.zeros_like(sc.coords)
    loss = api.backward(sc.coords, g, sc.assign, sc.gt_pose, *loss_args, *sc.params)
    hy = api.last_hypotheses(losses=True)
    contrib = np.asarray(bt.probs) >= O.PROB_THRESH
    assert np.abs(hy["scores"] - np.array(bt.scores)).max() < tol
    assert api.last_stats()["n_contrib"] == int(contrib.sum())
    assert np.abs(hy["losses"] - np.array(bt.losses)).max() < 1e-5 * max(1.0, np.abs(bt.losses).max())
    assert abs(loss - l_ref) < 1e-6 * max(1.0, abs(l_ref))
    if name == "tight_cut":       # most contributing hypotheses take the sqrt(cut * loss) branch
        assert (np.asarray(bt.losses)[contrib] > loss_args[2]).mean() > 0.5
    rep = GT.assert_classwise(g, g_ref, GT.cell_classes(sc.coords.shape, sc.assign, bt), BAR_SCENES, name)
    print(f"{name}: {GT.fmt(rep)}")


# ---- the hypotheses node and the stream-ordered calls at one non-default set ------------------------------------------
NODE_SET = "unfolded_alpha1000"


def test_reference_loss_through_the_node_is_esac_backward(api):
    import torch
    from esac_b200.autograd import esac_hypotheses, reference_pose_loss
    sc, w, seed = backward_scene(NODE_SET)
    coords = torch.from_numpy(sc.coords).cuda().requires_grad_(True)
    api.set_seed(seed)
    scores, poses, contrib = esac_hypotheses(coords, torch.from_numpy(sc.assign).cuda(), *sc.params)
    losses = reference_pose_loss(poses, torch.from_numpy(sc.gt_pose).cuda(), *w)
    L = (torch.softmax(scores, 0) * losses).sum()
    L.backward()
    api.set_seed(seed)
    g_ref = np.zeros_like(sc.coords)
    l_ref = api.backward(sc.coords, g_ref, sc.assign, sc.gt_pose, *w, *sc.params)
    hy = api.last_hypotheses(losses=True)
    assert np.array_equal(poses.detach().cpu().numpy(), hy["refined"])
    assert np.array_equal(scores.detach().cpu().numpy(), hy["scores"])
    assert int(contrib.sum()) == api.last_stats()["n_contrib"] >= 1
    assert abs(L.item() - l_ref) <= 1e-12 * abs(l_ref), (L.item(), l_ref)
    g = coords.grad.cpu().numpy()
    scale = np.abs(g_ref).max()
    assert scale > 0 and np.abs(g - g_ref).max() <= 1e-6 * scale


@pytest.fixture
def own_context(api):
    """A context of its own: the stream-ordered workspace of the shared one may be pinned by an earlier capture."""
    import torch
    dev = torch.cuda.current_device()
    saved = api._contexts.get(dev)
    ctx = api.Context(dev)
    api._contexts[dev] = ctx
    ctx.set_option("fixed_seed", 1)
    try:
        yield ctx
    finally:
        torch.cuda.synchronize()
        if saved is not None:
            api._contexts[dev] = saved
        else:
            api._contexts.pop(dev, None)
        ctx.close()


def _capture(fn):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def test_captured_node_and_backward_equal_eager_bitwise(api, own_context):
    """A tape written at tau 6, alpha 1000, beta 2 and maxReproj 100: the captured hypotheses_forward_async +
    hypotheses_backward_async read them back from the tape header, and must give the eager node's scores, poses and
    gradients bit for bit; the captured backward_async at the same values must give esac.backward's loss and gradient."""
    import torch
    sc, w, seed = backward_scene(NODE_SET)
    E, _, H, W = sc.coords.shape
    M = len(sc.assign)
    z = dict(device="cuda")
    tail = (sc.tau, sc.alpha, sc.beta, sc.max_reproj)
    rng = np.random.default_rng(5)
    d_scores = torch.from_numpy(rng.standard_normal(M)).cuda()
    d_poses = torch.from_numpy(rng.standard_normal((M, 6))).cuda()
    g0 = torch.from_numpy((rng.standard_normal(sc.coords.shape) * 1e-3).astype(np.float32)).cuda()
    coords = torch.from_numpy(sc.coords).cuda()
    assign = torch.from_numpy(sc.assign).cuda()
    shifts = torch.tensor([[sc.shiftX, sc.shiftY]], dtype=torch.int32, **z)
    cams = torch.tensor([[sc.f, sc.ppx, sc.ppy]], **z)
    gt = torch.from_numpy(sc.gt_pose).cuda()
    # eager
    api.set_seed(seed)
    e_scores, e_poses, e_contrib, tape = api.hypotheses_forward(coords, assign, *sc.params)
    e_grads = g0.clone()
    api.hypotheses_backward(tape, coords, e_grads, d_scores, d_poses)
    api.set_seed(seed)
    b_grads = g0.clone()
    b_loss = api.backward(coords, b_grads, assign, gt, *w, *sc.params)
    # captured
    api.reserve_backward_async(1, E, H, W, M, sc.sub)
    tapes = torch.zeros(api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, **z)
    scores, poses = torch.zeros(1, M, dtype=torch.float64, **z), torch.zeros(1, M, 6, dtype=torch.float64, **z)
    contrib = torch.zeros(1, M, dtype=torch.bool, **z)
    fst, bst, lst = (torch.full((1,), 7, dtype=torch.int32, **z) for _ in range(3))
    grads, bgrads = torch.zeros(1, E, 3, H, W, **z), torch.zeros(1, E, 3, H, W, **z)
    losses = torch.zeros(1, dtype=torch.float64, **z)
    c1, a1, gt1 = coords[None].contiguous(), assign[None].contiguous(), gt[None].contiguous()

    def node():
        api.hypotheses_forward_async(c1, a1, shifts, cams, *tail, sc.sub, tapes, scores, poses, contrib, fst)
        api.hypotheses_backward_async(tapes, c1, grads, M, d_scores[None].contiguous(), d_poses[None].contiguous(), bst)

    def bwd():
        api.backward_async(c1, bgrads, a1, gt1, shifts, cams, *w, *tail, sc.sub, losses, lst)

    gn, gb = _capture(node), _capture(bwd)
    grads.copy_(g0[None])
    bgrads.copy_(g0[None])
    api.set_seed(seed)
    gn.replay()
    api.set_seed(seed)
    gb.replay()
    torch.cuda.synchronize()
    assert int(fst[0]) == 0 and int(bst[0]) == 0 and int(lst[0]) == 0, (fst, bst, lst)
    np.testing.assert_array_equal(scores[0].cpu().numpy(), e_scores.cpu().numpy())
    np.testing.assert_array_equal(poses[0].cpu().numpy(), e_poses.cpu().numpy())
    np.testing.assert_array_equal(contrib[0].cpu().numpy(), e_contrib.cpu().numpy())
    np.testing.assert_array_equal(grads[0].cpu().numpy(), e_grads.cpu().numpy())
    assert np.float64(losses[0].item()) == np.float64(b_loss)
    np.testing.assert_array_equal(bgrads[0].cpu().numpy(), b_grads.cpu().numpy())
    assert bool(e_contrib.any()) and float((e_grads - g0).abs().max()) > 0
