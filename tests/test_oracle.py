"""The oracle itself (CPU): known answers, internal consistency, and the C restatement against the cv2 one.

The reference ships no golden vectors (SURVEY.md section 4), so the oracle is pinned by (i) executing real
OpenCV for every primitive, (ii) exact recovery of a known pose, (iii) agreement of two independent
restatements (Python/cv2 and C without OpenCV) of the scoring stage, (iv) committed golden fixtures generated
by the oracle (tests/golden/) that guard against silent drift."""
from pathlib import Path

import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error
from oracle import esac_oracle as O
from oracle.build import c_score

GOLD = Path(__file__).resolve().parent / "golden"


def test_forward_recovers_known_pose_noise_free():
    sc = make_scene(E=1, H=24, W=32, M=8, sub=8, seed=2, outlier_frac=0.0, noise=0.0)
    out = np.zeros((4, 4), np.float32)
    e, tr = O.forward(sc.coords, sc.assign, out, *sc.params, seed=3, trace=True)
    rot, trans = pose_error(out, sc.gt_pose)
    assert e == 0 and rot < 1e-3 and trans < 1e-4
    assert tr.scores[tr.winner] > 90  # nearly every cell is an inlier (alpha = 100)


def test_forward_with_outliers_picks_gt_expert():
    sc = make_scene(E=3, H=24, W=32, M=24, sub=8, seed=5)
    out = np.zeros((4, 4), np.float32)
    e = O.forward(sc.coords, sc.assign, out, *sc.params, seed=1)
    rot, trans = pose_error(out, sc.gt_pose)
    assert e == sc.gt_expert and rot < 1.0 and trans < 0.05


def test_sampling_never_uses_last_row_or_column():
    """irand(0, imW-1) -> uniform_int(0, imW-2): esac_util.h:167-168 + thread_rand.cpp:68-71."""
    W, H = 7, 5
    xs, ys = set(), set()
    for h in range(20):
        for t in range(20):
            for (x, y) in O.draw_minimal_set(9, h, t, W, H):
                xs.add(x); ys.add(y)
    assert max(xs) == W - 2 and max(ys) == H - 2 and min(xs) == 0 and min(ys) == 0


@pytest.mark.parametrize("kw", [{}, {"shiftX": 3, "shiftY": -2}, {"world_offset": 500.0}])
def test_c_restatement_matches_cv2_oracle_scores(kw):
    sc = make_scene(E=2, H=24, W=31, M=12, sub=8, seed=7, **kw)
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    samp = O.create_sampling(31, 24, sc.sub, sc.shiftX, sc.shiftY)
    hyps = O.sample_hypotheses(sc.coords, sc.assign, samp, K, 10000, sc.tau, 5)
    errs = [O.get_repro_errs(sc.coords, h.rvec, h.tvec, int(sc.assign[i]), samp, K, sc.max_reproj)[0] for i, h in enumerate(hyps)]
    ref = np.array(O.get_hyp_scores(errs, sc.tau, sc.alpha, sc.beta))
    p6 = np.array([np.concatenate([h.rvec.ravel(), h.tvec.ravel()]) for h in hyps])
    got, _ = c_score(sc.coords, sc.assign, p6, *sc.params)
    assert np.abs(got - ref).max() < 1e-10


def _score_pin_poses(sc, seed):
    """Sampled hypotheses (near the truth on the ground-truth plane) followed by arbitrary poses (cells behind the camera,
    far off the image): every branch of the projection and the clamp."""
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    H, W = sc.coords.shape[2:]
    samp = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY)
    hyps = O.sample_hypotheses(sc.coords, sc.assign, samp, K, 10000, sc.tau, seed)
    p6 = np.array([np.concatenate([h.rvec.ravel(), h.tvec.ravel()]) for h in hyps])
    rng = np.random.default_rng(seed)
    k = len(p6) // 3
    p6[-k:, :3] = rng.normal(0, 0.5, (k, 3))
    p6[-k:, 3:] = p6[-k:, 3:] + rng.normal(0, 2.0, (k, 3)) * (1.0 + np.abs(p6[-k:, 3:]).max(axis=1, keepdims=True) * 1e-2)
    return K, samp, p6


@pytest.mark.parametrize("kw", [
    dict(E=2, H=24, W=31, M=12, sub=8, seed=7),
    dict(E=2, H=21, W=29, M=12, sub=3, seed=8, shiftX=-4, shiftY=-7),           # odd sub-sampling, negative shifts
    dict(E=3, H=20, W=26, M=15, sub=4, seed=9, shiftX=3, shiftY=-5, world_offset=700.0),
    dict(E=1, H=16, W=20, M=9, sub=8, seed=10, outdoor=True, unit_scale=1000.0),  # world scale in millimetres
])
def test_fp64_score_reference_matches_both_oracles(kw):
    """oracle/score_fp64.py (the reference the GPU launch-shape tests compare with) against the cv2 oracle and the C
    restatement: the scores agree to 1e-5, and so does every cell's soft-inlier weight wherever cv2's float32 error is not
    within float rounding of maxReproj (there the fp64 clamp and the float one may fall on different sides)."""
    from oracle import score_fp64
    sc = make_scene(**kw)
    K, samp, p6 = _score_pin_poses(sc, kw["seed"])
    ref64, w64 = score_fp64.score(sc.coords, sc.assign, p6, *sc.params)
    errs = [O.get_repro_errs(sc.coords, p[:3].reshape(3, 1), p[3:].reshape(3, 1), int(sc.assign[i]), samp, K, sc.max_reproj)[0]
            for i, p in enumerate(p6)]
    cv = np.array(O.get_hyp_scores(errs, sc.tau, sc.alpha, sc.beta))
    cs, _ = c_score(sc.coords, sc.assign, p6, *sc.params)
    assert np.isfinite(cv).all()
    assert np.abs(ref64 - cv).max() < 1e-5, np.abs(ref64 - cv).max()
    assert np.abs(ref64 - cs).max() < 1e-5, np.abs(ref64 - cs).max()
    e32 = np.stack(errs).astype(np.float64)
    w_cv = score_fp64.soft_inlier_weights(e32, sc.tau, sc.beta)
    ok = np.isfinite(e32) & (np.abs(e32 - sc.max_reproj) > 1e-3)
    assert ok.sum() >= 0.2 * ok.size and (e32[ok] < sc.tau).sum() >= 10    # the comparison covers inliers as well as outliers
    assert np.abs(w64[ok] - w_cv[ok]).max() < 1e-5, np.abs(w64[ok] - w_cv[ok]).max()


def test_fp64_score_reference_rules_for_degenerate_cells():
    """A cell at depth exactly 0 projects with z = 1 (OpenCV's `z ? 1/z : 1`); a non-finite cell counts as maxReproj."""
    from oracle import score_fp64
    coords = np.zeros((1, 3, 2, 3), np.float32)
    coords[0, :, 0, 1] = [0.01, -0.02, 0.0]            # camera frame (identity pose): z = 0 -> projects to pp + f (x, y)
    coords[0, :, 1, 0] = [np.nan, 0.0, 1.0]
    coords[0, :, 1, 1] = [0.0, 0.0, -2.0]              # behind the camera, on the optical axis: the principal point
    coords[0, 2, 0, 0] = coords[0, 2, 0, 2] = coords[0, 2, 1, 2] = 1.0
    f, ppx, ppy, sub = 100.0, 7.0, 5.0, 3
    errs = score_fp64.repro_errs(coords, [0], np.zeros((1, 6)), 0, 0, f, ppx, ppy, 100.0, sub)[0]
    px, py = score_fp64.pixel_centres(2, 3, sub, 0, 0)
    assert px[0].tolist() == [1, 4, 7] and py[:, 0].tolist() == [1, 4]
    assert errs[0, 1] == pytest.approx(np.hypot(ppx + f * 0.01 - 4, ppy - f * 0.02 - 1), abs=1e-12)
    assert errs[1, 0] == 100.0
    assert errs[1, 1] == pytest.approx(np.hypot(ppx - 4, ppy - 4), abs=1e-12)
    w = score_fp64.soft_inlier_weights(np.array([-1e9, 10.0, 1e9]), 10.0, 0.5)
    assert w.tolist() == [1.0, 0.5, 0.0]


def test_softmax_entropy_draw():
    p = O.softmax([1.0, 3.0, 3.0, 2.0])
    assert abs(p.sum() - 1) < 1e-15 and O.draw(p) == 1  # first strict maximum
    assert abs(O.entropy([0.5, 0.5]) - 1.0) < 1e-15
    assert O.entropy([1.0, 0.0]) == 0.0


def test_loss_cut_and_clamp():
    T = np.eye(4)
    T2 = np.eye(4); T2[:3, 3] = [3.0, 0, 0]
    assert abs(O.loss(T, T2, 1.0, 100.0, 1e9) - 300.0) < 1e-9
    assert abs(O.loss(T, T2, 1.0, 100.0, 100.0) - np.sqrt(100.0 * 300.0)) < 1e-9


def test_backward_accumulates_and_only_touches_assigned_experts():
    sc = make_scene(E=3, H=16, W=20, M=12, sub=8, seed=11)
    g = np.full_like(sc.coords, 0.25)
    loss, bt = O.backward(sc.coords, g, sc.assign, sc.gt_pose, 1.0, 100.0, 100.0, *sc.params, seed=2, trace=True)
    assert loss > 0 and np.isfinite(g).all()
    used = set(int(sc.assign[h]) for h in range(len(sc.assign)) if bt.probs[h] >= O.PROB_THRESH)
    for e in range(3):
        if e not in used:
            assert np.all(g[e] == 0.25)
    assert any(np.any(g[e] != 0.25) for e in used)


def test_golden_fixtures_still_reproduce():
    """tests/golden/*.npz (other than ref_*) were written by tests/golden/make_golden.py from this oracle."""
    files = sorted(p for p in GOLD.glob("*.npz") if not p.name.startswith("ref_"))
    assert files, "run python tests/golden/make_golden.py"
    for f in files:
        z = np.load(f)
        out = np.zeros((4, 4), np.float32)
        params = tuple(z["params"].tolist())
        params = (int(params[0]), int(params[1])) + tuple(float(v) for v in params[2:9]) + (int(params[9]),)
        e, tr = O.forward(z["coords"], z["assign"], out, *params, seed=int(z["seed"]), trace=True)
        assert e == int(z["expert"])
        assert np.abs(np.array(tr.scores) - z["scores"]).max() < 1e-9
        assert np.abs(out - z["pose"]).max() < 1e-6


def test_direct_score_gradient_matches_finite_differences():
    """Pins the one part of the reference's gradient that IS an exact derivative: d score / d sceneCoordinates at a fixed
    pose (dScore's direct term, esac_derivative.h:258-306) against central differences of an fp64 restatement of the score
    (differences through cv2.projectPoints are useless: its float output quantises at ~3e-5 px, SURVEY.md Appendix A).
    The other terms cannot be pinned this way: path I (esac.cpp:373-463) linearises the *norms* of the residuals, which
    drops a curvature term of the same size as the one it keeps, so the reference's gradient is not the gradient of its own
    expected loss (measured: finite differences of the refined pose disagree with -(J^T J)^-1 J^T dNdO in sign and size)."""
    import cv2
    sc = make_scene(E=1, H=8, W=10, M=6, sub=8, seed=1, outlier_frac=0.0, noise=0.01)
    H, W = 8, 10
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    samp = O.create_sampling(W, H, sc.sub, 0, 0)
    hyps = O.sample_hypotheses(sc.coords, sc.assign, samp, K, 10000, sc.tau, 5)
    rng = np.random.default_rng(0)
    d = rng.normal(size=sc.coords.shape).astype(np.float32)
    eps = 5e-4
    cp, cm = (sc.coords + eps * d).astype(np.float32), (sc.coords - eps * d).astype(np.float32)

    def score64(c, rv, tv):
        R, _ = cv2.Rodrigues(rv)
        xc = c[0].reshape(3, -1).T.astype(np.float64) @ R.T + tv.ravel()
        u = xc[:, 0] / xc[:, 2] * sc.f + sc.ppx
        v = xc[:, 1] / xc[:, 2] * sc.f + sc.ppy
        px = samp[:, :, 0].reshape(-1).astype(np.float64)
        py = samp[:, :, 1].reshape(-1).astype(np.float64)
        err = np.minimum(np.sqrt((u - px) ** 2 + (v - py) ** 2), sc.max_reproj)
        return (sc.alpha / (H * W)) * np.sum(1 - 1 / (1 + np.exp(-sc.beta * (err - sc.tau))))

    fd, an = [], []
    pts3, pts2 = O._collect(sc.coords, 0, samp)
    dcol = d[0].transpose(2, 1, 0).reshape(W * H, 3)
    for hy in hyps:
        fd.append((score64(cp, hy.rvec, hy.tvec) - score64(cm, hy.rvec, hy.tvec)) / (2 * eps))
        err = O.get_repro_errs(sc.coords, hy.rvec, hy.tvec, 0, samp, K, sc.max_reproj)[0]
        st = 1 / (1 + np.exp(-(sc.beta * (err.astype(np.float64) - sc.tau))))
        w = -st * (1 - st) * sc.beta * (sc.alpha / (H * W))
        R, _ = cv2.Rodrigues(hy.rvec)
        dP = O.d_project_d_obj_batch(pts2, pts3, R, hy.tvec, K, sc.max_reproj) * w.T.reshape(-1)[:, None]
        an.append(float((dP * dcol).sum()))
    fd, an = np.array(fd), np.array(an)
    assert np.corrcoef(fd, an)[0, 1] > 0.995
    assert np.abs(fd - an).max() < 0.05 * np.abs(fd).max()


def test_assign_hypotheses_follows_the_callers_semantics():
    """clamp_probs / multinomial(replacement) / histc as train_esac.py:130-140 runs them, checked against torch."""
    import torch
    rng = np.random.default_rng(5)
    w = rng.random((3, 9)).astype(np.float32)
    w[0, 4] = 0.0
    # util.clamp_probs restated with torch.sort exactly as the caller does (util.py:43-48)
    for n in (-1, 0, 2, 9, 20):
        t = torch.from_numpy(w[1].copy())
        if n >= 0:
            s_prob, s_indx = t.sort(dim=0, stable=True)
            for i, idx in enumerate(s_indx):
                if i < s_prob.size(0) - n:
                    t[idx] = 0
        assert np.array_equal(O.clamp_probs(w[1], n), t.numpy())
    a, h = O.assign_hypotheses(w, 4000, seed=11)
    assert a.shape == (3, 4000) and a.dtype == np.int64
    for b in range(3):
        ref_hist = torch.histc(torch.from_numpy(a[b]).float(), bins=9, min=0, max=8).numpy()
        assert np.array_equal(h[b], ref_hist)
        p = w[b] / w[b].sum()
        assert np.abs(h[b] / 4000 - p).max() < 0.03          # ~4 sigma of a binomial proportion
    assert h[0, 4] == 0                                       # zero weight is never drawn
    a2, h2 = O.assign_hypotheses(w, 50, seed=11, keep_top=2)
    for b in range(3):
        top2 = set(np.argsort(w[b], kind="stable")[-2:].tolist())
        assert set(np.unique(a2[b]).tolist()) <= top2
    a3, h3 = O.assign_hypotheses(w, 16, seed=11, single=True)
    assert all(len(np.unique(a3[b])) == 1 for b in range(3)) and np.all(h3.sum(axis=1) == 16)
    assert np.array_equal(a3[:, 0], a[:, 0])                  # the single draw is draw 0 of the stream
    with pytest.raises(RuntimeError):
        O.assign_hypotheses(np.zeros((1, 4), np.float32), 4, seed=1)
    with pytest.raises(RuntimeError):
        O.assign_hypotheses(np.array([[0.5, -0.1]], np.float32), 4, seed=1)


def test_reproj_loss_oracle_gradient_matches_closed_form():
    """The torch restatement of ref_expert.py:103-148 (autograd) against an independent numpy closed form in float64."""
    import torch
    from oracle.reproj_loss_oracle import reproj_loss_and_grad
    sc = make_scene(E=1, H=12, W=15, M=8, sub=8, seed=21, outlier_frac=0.3)
    f, padx, pady, cut = 525.0, 3, -2, 10.0
    X = sc.coords[0].astype(np.float64)
    X[:, 0, 0] = [0.0, 0.0, -50.0]                       # a point behind the camera: depth clamp branch
    loss, g = reproj_loss_and_grad(torch.from_numpy(X), torch.from_numpy(sc.gt_pose.astype(np.float64)), f, padx, pady, cut,
                                   dtype=torch.float64)
    Tinv = np.linalg.inv(sc.gt_pose.astype(np.float64))[:3]
    H, W = X.shape[1:]
    cx, cy = W * 8 / 2, H * 8 / 2
    total = 0.0
    G = np.zeros_like(X)
    for y in range(H):
        for x in range(W):
            c = Tinv[:, :3] @ X[:, y, x] + Tinv[:, 3]
            nu, nv = f * c[0] + cx * c[2], f * c[1] + cy * c[2]
            open_ = c[2] >= 0.1
            z = c[2] if open_ else 0.1
            du, dv = nu / z - (x * 8 + 4.0 - padx), nv / z - (y * 8 + 4.0 - pady)
            err = np.hypot(du, dv)
            e = min(err, 100.0)
            total += e if e <= cut else np.sqrt(cut * e)
            gl = 0.0 if err > 100.0 else (1.0 if e <= cut else 0.5 * cut / np.sqrt(cut * e))
            gu, gv = gl * du / err, gl * dv / err
            gc = np.array([gu * f / z, gv * f / z, (gu * cx + gv * cy) / z - ((gu * nu + gv * nv) / z ** 2 if open_ else 0.0)])
            G[:, y, x] = Tinv[:, :3].T @ gc / (H * W)
    assert abs(loss - total / (H * W)) < 1e-12 * max(1.0, abs(loss))
    assert np.abs(g.numpy() - G).max() < 1e-12 * max(1.0, np.abs(G).max())


# ---- the oracle against outputs of the reference's own compiled code (tests/golden/ref_*.npz) -------------------------
def _ref_fixtures_small():
    from ref_golden_util import REF_GOLD
    return [p for p in REF_GOLD if "coords" in np.load(p).files]


@pytest.mark.parametrize("path", _ref_fixtures_small(), ids=lambda p: p.stem)
def test_oracle_reproduces_the_compiled_reference_fixtures(path):
    """No reference checkout needed: the fixtures were written by oracle/_ref (unmodified esac.cpp on the real OpenCV, single
    thread, default mt19937 stream); ThreadRandStream replays that stream."""
    from ref_golden_util import params_of
    z = np.load(path)
    params = params_of(z)
    out = np.zeros((4, 4), np.float32)
    e, tr = O.forward(z["coords"], z["assign"], out, *params, mt=O.ThreadRandStream(1305), trace=True)
    assert e == int(z["expert"])
    assert np.abs(out - z["pose"]).max() <= 1e-6
    assert [h.tries for h in tr.hyps] == z["tries"].tolist()
    assert [[list(c) for c in h.cells] for h in tr.hyps] == z["cells"][:, -1].tolist()
    g = np.zeros_like(z["coords"])
    w_rot, w_trans, cut = (float(v) for v in z["loss_args"])
    loss, bt = O.backward(z["coords"], g, z["assign"], z["gt_pose"], w_rot, w_trans, cut, *params, mt=O.ThreadRandStream(1305),
                          trace=True)
    assert abs(loss - float(z["loss"])) <= 1e-9 * max(1.0, abs(float(z["loss"])))
    assert np.abs(g - z["grads"]).max() <= 1e-6 * np.abs(z["grads"]).max()
    if "clamped_jr" in z.files:  # the "clamping for stability" fixtures (esac.cpp:436-437, esac_derivative.h:287)
        assert bt.clamped_jr == z["clamped_jr"].tolist() and bt.clamped_dpnp == z["clamped_dpnp"].tolist()


def test_clamp_fixtures_really_trip_the_clamps():
    """The reference's gradient on these fixtures is only reproduced WITH the two `> 10` clamps: without them the oracle's
    gradient moves by far more than the parity tolerance (1e-3 of the largest entry), so an implementation that matches the
    fixtures provably clamps where the reference does.  The J_R pair brackets the threshold: same scene in units of 1/7000 m
    (every contributing hypothesis clamped, path I vanishes) and 1/5000 m (none clamped)."""
    from ref_golden_util import GOLD_DIR, params_of
    seen = {}
    for name in ("ref_clamp_dpnp_9x12", "ref_clamp_jr_on_12x16", "ref_clamp_jr_off_12x16"):
        z = np.load(GOLD_DIR / f"{name}.npz")
        seen[name] = z
        g_ref = z["grads"]
        g_no = np.zeros_like(g_ref)
        w_rot, w_trans, cut = (float(v) for v in z["loss_args"])
        O.backward(z["coords"], g_no, z["assign"], z["gt_pose"], w_rot, w_trans, cut, *params_of(z), mt=O.ThreadRandStream(1305),
                   clamp_thresh=np.inf)
        moved = np.abs(g_no - g_ref).max() / np.abs(g_ref).max()
        if name == "ref_clamp_jr_off_12x16":
            assert len(z["clamped_jr"]) == 0
        else:
            assert moved > 0.05, (name, moved)
    assert len(seen["ref_clamp_dpnp_9x12"]["clamped_dpnp"]) == 9 and len(seen["ref_clamp_dpnp_9x12"]["clamped_jr"]) == 0
    assert len(seen["ref_clamp_jr_on_12x16"]["clamped_jr"]) == 3
    # the clamp removes path I altogether: the gradient collapses by four orders of magnitude between the two unit scales
    assert np.abs(seen["ref_clamp_jr_on_12x16"]["grads"]).max() < 1e-3 * np.abs(seen["ref_clamp_jr_off_12x16"]["grads"]).max()
