"""GPU parity of the forward path against the cv2 oracle (run with `-m gpu` on an H100).

Tolerances are BASELINE.json's: 1e-4 on soft-inlier scores, 1e-3 deg / 1e-3 cm on the final pose."""
import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-4
ROT_TOL_DEG = 1e-3
TRANS_TOL_M = 1e-5  # 1e-3 cm


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


def _oracle_hyps(sc, seed):
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    H, W = sc.coords.shape[2:]
    sampling = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY)
    hyps = O.sample_hypotheses(sc.coords, sc.assign, sampling, K, O.MAX_SAMPLING_TRIES, sc.tau, seed)
    return K, sampling, hyps


@pytest.mark.parametrize("E,H,W,M,sub,kw", [
    (1, 60, 80, 64, 8, {}),                                  # config 1 shape (DSAC++ mode)
    (3, 30, 40, 48, 8, {"shiftX": 3, "shiftY": -4}),          # shifted sampling grid (training augmentation)
    (2, 60, 107, 32, 8, {}),                                  # N = 6420: N % 4 == 0, vector loads (ppt 2), ragged tile
    (2, 37, 53, 32, 4, {}),                                   # odd sizes
    (2, 24, 32, 40, 8, {"world_offset": 700.0}),              # world-scale coordinates (re-centring path)
    (2, 61, 107, 32, 8, {}),                                  # N = 6527 odd -> scalar load path, ragged tile
])
def test_scores_match_oracle_for_given_poses(api, E, H, W, M, sub, kw):
    sc = make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=11, **kw)
    K, sampling, hyps = _oracle_hyps(sc, 5)
    errs = [O.get_repro_errs(sc.coords, hy.rvec, hy.tvec, int(sc.assign[h]), sampling, K, sc.max_reproj)[0]
            for h, hy in enumerate(hyps)]
    ref = np.array(O.get_hyp_scores(errs, sc.tau, sc.alpha, sc.beta))
    poses6 = np.array([np.concatenate([hy.rvec.ravel(), hy.tvec.ravel()]) for hy in hyps])
    got = api.score_poses(sc.coords, sc.assign, poses6, *sc.params)
    assert np.abs(got - ref).max() < SCORE_TOL, (np.abs(got - ref).max(), ref[:4], got[:4])


def test_scores_behind_camera_and_clamped(api):
    """Cells behind the camera mirror through the principal point (no cheirality test in the reference)
    and errors clamp at maxReproj."""
    sc = make_scene(E=1, H=30, W=40, M=8, sub=8, seed=3)
    rng = np.random.default_rng(0)
    poses6 = np.zeros((8, 6))
    poses6[:, :3] = rng.normal(0, 0.5, (8, 3))
    poses6[:, 3:] = rng.normal(0, 2.0, (8, 3))  # arbitrary poses: many cells behind the camera / far off
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    sampling = O.create_sampling(40, 30, sc.sub, 0, 0)
    errs = [O.get_repro_errs(sc.coords, p[:3].reshape(3, 1), p[3:].reshape(3, 1), 0, sampling, K, sc.max_reproj)[0]
            for p in poses6]
    ref = np.array(O.get_hyp_scores(errs, sc.tau, sc.alpha, sc.beta))
    got = api.score_poses(sc.coords, sc.assign, poses6, *sc.params)
    assert np.abs(got - ref).max() < SCORE_TOL


@pytest.mark.parametrize("E,H,W,M", [(1, 60, 80, 64), (4, 30, 40, 64)])
def test_sampling_matches_oracle_stream(api, E, H, W, M):
    """Same counter stream -> same accepted minimal sets, same try counts, same P3P poses."""
    sc = make_scene(E=E, H=H, W=W, M=M, sub=8, seed=21)
    _, _, hyps = _oracle_hyps(sc, 77)
    api.set_seed(77)
    out = np.zeros((4, 4), np.float32)
    api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    assert [h.tries for h in hyps] == hy["tries"].tolist()
    assert [[list(c) for c in h.cells] for h in hyps] == hy["cells"].tolist()
    ref = np.array([np.concatenate([h.rvec.ravel(), h.tvec.ravel()]) for h in hyps])
    assert np.abs(ref - hy["poses"]).max() < 1e-8


@pytest.mark.parametrize("seed,E,H,W,M,sub,kw", [
    (1, 1, 60, 80, 64, 8, {}),
    (2, 3, 30, 40, 64, 8, {}),
    (3, 7, 60, 80, 256, 8, {}),                       # config 2 at the native shape
    (4, 2, 60, 107, 64, 8, {"shiftX": -2, "shiftY": 4}),
    (5, 2, 45, 60, 64, 8, {"outlier_frac": 0.7}),
    (6, 2, 41, 53, 64, 3, {"shiftX": 2, "shiftY": -1}),  # odd sub-sampling: pixel centre x*3 + 1
])
def test_forward_matches_oracle(api, seed, E, H, W, M, sub, kw):
    sc = make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=seed, **kw)
    ref_pose = np.zeros((4, 4), np.float32)
    ref_e, tr = O.forward(sc.coords, sc.assign, ref_pose, *sc.params, seed=100 + seed, trace=True)
    api.set_seed(100 + seed)
    out = np.zeros((4, 4), np.float32)
    e = api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    st = api.last_stats()
    assert np.abs(hy["scores"] - np.array(tr.scores)).max() < SCORE_TOL
    # winner: identical unless the two best scores are closer than the score tolerance (SURVEY hard part 4)
    s = np.sort(np.array(tr.scores))[::-1]
    if len(s) == 1 or s[0] - s[1] > 10 * SCORE_TOL:
        assert st["winner"] == tr.winner and e == ref_e
        assert st["refine_rounds"] == tr.rounds
        rot, trans = pose_error(out, ref_pose)
        assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (rot, trans)
        # the same comparison before the float32 rounding of outPose
        ref6 = hy["refined"][tr.winner]
        Ta = O.pose2trans(tr.ref_rvec, tr.ref_tvec)
        Tb = O.pose2trans(ref6[:3].reshape(3, 1), ref6[3:].reshape(3, 1))
        rot, trans = pose_error(Tb, Ta)
        assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (rot, trans)
    assert abs(st["entropy"] - tr.entropy) < 1e-3


def test_forward_cuda_tensors_and_stride0_assignment(api):
    import torch
    sc = make_scene(E=2, H=30, W=40, M=32, sub=8, seed=9)
    coords = torch.from_numpy(sc.coords)
    expert = torch.tensor([sc.gt_expert], dtype=torch.int64)
    assign = expert.expand(32)  # stride-0 view, as test_esac.py:173 builds it
    assert assign.stride(0) == 0
    api.set_seed(5)
    out_cpu = torch.zeros(4, 4)
    e1 = api.forward(coords, assign, out_cpu, *sc.params)
    api.set_seed(5)
    out_gpu = torch.zeros(4, 4, device="cuda")
    e2 = api.forward(coords.cuda(), assign.cuda(), out_gpu, *sc.params)
    assert e1 == e2 == sc.gt_expert
    assert torch.equal(out_cpu, out_gpu.cpu())
    rot, trans = pose_error(out_cpu.numpy(), sc.gt_pose)
    assert rot < 1.0 and trans < 0.05


def test_forward_is_ordered_after_pending_work_on_torchs_stream(api):
    """A caller hands over expert outputs that are still being produced on torch's current stream (train_esac.py computes
    `prediction` right before the call): the library must queue behind that work, on the default stream and on a side stream."""
    import torch
    sc = make_scene(E=2, H=30, W=40, M=32, sub=8, seed=9)
    coords = torch.from_numpy(sc.coords).cuda()
    assign = torch.from_numpy(sc.assign).cuda()
    api.set_seed(5)
    ref = torch.zeros(4, 4, device="cuda")
    e_ref = api.forward(coords, assign, ref, *sc.params)
    big = torch.randn(4096, 4096, device="cuda")
    for stream in (None, torch.cuda.Stream()):
        with torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.default_stream()):
            late = torch.zeros_like(coords)
            late_assign = torch.full_like(assign, 10 ** 6)          # poison: flagged as a bad expert index if read early
            torch.cuda.synchronize()
            for _ in range(40):                                     # ~10 ms of queued work ahead of the real inputs
                big = big @ big * 1e-3
            late.copy_(coords, non_blocking=True)
            late_assign.copy_(assign, non_blocking=True)
            api.set_seed(5)
            out = torch.zeros(4, 4, device="cuda")
            e = api.forward(late, late_assign, out, *sc.params)
        torch.cuda.synchronize()
        assert e == e_ref and torch.equal(out, ref)


def test_forward_known_answer_noise_free(api):
    """Noise-free map: the estimate must be the ground-truth pose."""
    sc = make_scene(E=1, H=30, W=40, M=16, sub=8, seed=4, outlier_frac=0.0, noise=0.0)
    out = np.zeros((4, 4), np.float32)
    api.set_seed(1)
    api.forward(sc.coords, sc.assign, out, *sc.params)
    rot, trans = pose_error(out, sc.gt_pose)
    assert rot < 1e-3 and trans < 1e-4  # limited by float32 coordinates


def test_refine_matches_oracle(api):
    sc = make_scene(E=2, H=60, W=80, M=24, sub=8, seed=6)
    K, sampling, hyps = _oracle_hyps(sc, 9)
    poses6 = np.array([np.concatenate([h.rvec.ravel(), h.tvec.ravel()]) for h in hyps])
    got, rounds, inl = api.refine_poses(sc.coords, sc.assign, poses6, sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy,
                                        sc.tau, sc.max_reproj, sc.sub)
    for h, hy in enumerate(hyps):
        errs, _ = O.get_repro_errs(sc.coords, hy.rvec, hy.tvec, int(sc.assign[h]), sampling, K, sc.max_reproj)
        r, t, im, rr = O.refine_hyp(sc.coords, errs, sampling, K, int(sc.assign[h]), sc.tau, O.MAX_REF_STEPS,
                                    sc.max_reproj, hy.rvec, hy.tvec)
        assert rr == rounds[h], (h, rr, rounds[h])
        assert (0 if im is None else int(im.sum())) == inl[h]
        Ta, Tb = O.pose2trans(r, t), O.pose2trans(got[h, :3].reshape(3, 1), got[h, 3:].reshape(3, 1))
        rot, trans = pose_error(Tb, Ta)
        assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (h, rot, trans)


@pytest.mark.parametrize("kw", [
    dict(E=2, H=60, W=80, M=24, sub=8, seed=6),                                                 # the reference's native shape
    dict(E=2, H=120, W=160, M=16, sub=4, seed=12, noise=0.05, outlier_frac=0.3),                # many errors close to tau
    dict(E=2, H=48, W=64, M=16, sub=8, seed=13, outdoor=True, world_offset=700.0),              # world-scale coordinates
    dict(E=1, H=24, W=32, M=12, sub=8, seed=14, unit_scale=7000.0, noise=0.002),                # lengths in 1/7000 m
    dict(E=1, H=30, W=40, M=12, sub=8, seed=15, shiftX=3, shiftY=-5, noise=0.1),                # shifted grid, heavy noise
])
def test_refinement_float_pretest_never_changes_a_decision(api, kw):
    """The inlier selection classifies clear cells with a float evaluation + rounding-error bound and runs getReproErrs'
    arithmetic only where in doubt (refine.cu lm_select): switching the pretest off must give bit-identical poses, rounds and
    inlier counts -- one differing cell would change the sums.  Start poses: ground truth perturbed, so every round moves."""
    sc = make_scene(**kw)
    rng = np.random.default_rng(kw["seed"])
    import cv2
    T = np.linalg.inv(sc.gt_pose.astype(np.float64))                     # scene (world -> camera) transform
    poses6 = np.zeros((len(sc.assign), 6))
    scale = float(kw.get("unit_scale", 1.0)) * (5.0 if kw.get("outdoor") else 1.0)
    for h in range(len(sc.assign)):                                      # a small motion IN THE CAMERA FRAME on top of the truth
        dR, _ = cv2.Rodrigues(rng.normal(0, 0.004, 3))
        R1 = dR @ T[:3, :3]
        t1 = dR @ T[:3, 3] + rng.normal(0, 0.02 * scale, 3)
        poses6[h, :3] = cv2.Rodrigues(R1)[0].ravel()
        poses6[h, 3:] = t1
    ctx = api.context()
    outs = []
    for pre in (0, 1):
        ctx.set_option("refine_pretest", pre)
        outs.append(api.refine_poses(sc.coords, sc.assign, poses6, sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy, sc.tau, sc.max_reproj, sc.sub))
    ctx.set_option("refine_pretest", 1)
    assert outs[0][2].tolist() == outs[1][2].tolist()          # inlier counts
    assert outs[0][1].tolist() == outs[1][1].tolist()          # accepted rounds
    assert np.array_equal(outs[0][0], outs[1][0])              # poses, bit for bit
    assert outs[0][2].max() >= 4 and outs[0][1].max() >= 1     # something was refined


def test_bad_arguments_raise(api):
    sc = make_scene(E=1, H=30, W=40, M=8, sub=8, seed=1)
    out = np.zeros((4, 4), np.float32)
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        api.forward(sc.coords.astype(np.float64), sc.assign, out, *sc.params)
    with pytest.raises(RuntimeError, match="expected scalar type Long"):
        api.forward(sc.coords, sc.assign.astype(np.int32), out, *sc.params)
    with pytest.raises(RuntimeError):
        api.forward(sc.coords, sc.assign + 5, out, *sc.params)  # expert index out of range


@pytest.mark.parametrize("kw", [dict(E=4, H=60, W=80, M=256, sub=8, seed=41, active_only=False, per_expert=True),
                                dict(E=2, H=120, W=160, M=128, sub=4, seed=42, outdoor=True, active_only=False, per_expert=True)])
def test_sampling_prefilter_does_not_change_results(api, kw):
    """The fp32 prefilter of the sampling waves may only drop tries the exact path rejects: with it switched off the
    accepted minimal sets, try counts and poses must be identical (hard maps: wrong experts need ~1e3 tries)."""
    sc = make_scene(**kw)
    out = np.zeros((4, 4), np.float32)
    res = []
    for flag in (1, 0):
        api.set_option("sample_prefilter", flag)
        api.set_seed(7)
        api.forward(sc.coords, sc.assign, out, *sc.params)
        res.append(api.last_hypotheses())
    api.set_option("sample_prefilter", 1)
    assert res[0]["tries"].max() > 500          # the scene did need many tries
    assert np.array_equal(res[0]["tries"], res[1]["tries"])
    assert np.array_equal(res[0]["cells"], res[1]["cells"])
    assert np.array_equal(res[0]["poses"], res[1]["poses"])


def test_forward_batch_equals_a_loop_of_forward(api):
    """BASELINE configs[2] shape of work (a batch of images): the batched entry must give what a loop of esac.forward
    gives (the call counter advances the sampling stream identically), for host and for CUDA tensors."""
    import torch
    B = 4
    scenes = [make_scene(E=3, H=30, W=40, M=48, sub=8, seed=60 + b) for b in range(B)]
    coords = np.stack([s.coords for s in scenes]); assign = np.stack([s.assign for s in scenes])
    api.set_option("fixed_seed", 0)
    try:
        api.set_seed(123)
        ref_e, ref_p = [], []
        for s in scenes:
            out = np.zeros((4, 4), np.float32)
            ref_e.append(api.forward(s.coords, s.assign, out, *scenes[0].params))
            ref_p.append(out)
        api.set_seed(123)
        outs = np.zeros((B, 4, 4), np.float32)
        e = api.forward_batch(coords, assign, outs, *scenes[0].params)
        assert e == ref_e and np.array_equal(outs, np.stack(ref_p))
        api.set_seed(123)
        outs_gpu = torch.zeros(B, 4, 4, device="cuda")
        e2 = api.forward_batch(torch.from_numpy(coords).cuda(), torch.from_numpy(assign).cuda(), outs_gpu, *scenes[0].params)
        assert e2 == ref_e and np.array_equal(outs_gpu.cpu().numpy(), np.stack(ref_p))
        api.set_seed(123)
        outs_pin = torch.zeros(B, 4, 4).pin_memory()
        e3 = api.forward_batch(torch.from_numpy(coords).pin_memory(), torch.from_numpy(assign), outs_pin, *scenes[0].params)
        assert e3 == ref_e and np.array_equal(outs_pin.numpy(), np.stack(ref_p))
    finally:
        api.set_option("fixed_seed", 1)
    assert [s.gt_expert for s in scenes] == ref_e


def test_tiny_problem_single_hypothesis(api):
    """M = 1, E = 1 on an 8x10 map: every reduction degenerates to one element."""
    sc = make_scene(E=1, H=8, W=10, M=1, sub=8, seed=13, outlier_frac=0.0, noise=0.0)
    ref = np.zeros((4, 4), np.float32)
    ref_e, tr = O.forward(sc.coords, sc.assign, ref, *sc.params, seed=3, trace=True)
    api.set_seed(3)
    out = np.zeros((4, 4), np.float32)
    e = api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    assert e == ref_e == 0 and hy["tries"].tolist() == [tr.hyps[0].tries]
    assert abs(hy["scores"][0] - tr.scores[0]) < 1e-4
    rot, trans = pose_error(out, ref)
    assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M


def test_many_experts_many_hypotheses(api):
    """E = 50 clusters (the reference's largest ensemble, environments/aachen) and M = 2048 on the native 60x80 map."""
    sc = make_scene(E=50, H=60, W=80, M=2048, sub=8, seed=14)
    api.set_seed(8)
    out = np.zeros((4, 4), np.float32)
    e = api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    assert e == sc.gt_expert and np.isfinite(hy["scores"]).all()
    # spot-check a handful of scores against the C oracle restatement
    from oracle.build import c_score
    idx = np.array([0, 1, 500, 1000, 2047])
    ref, _ = c_score(sc.coords, sc.assign[idx], hy["poses"][idx], *sc.params)
    assert np.abs(ref - hy["scores"][idx]).max() < SCORE_TOL
    rot, trans = pose_error(out, sc.gt_pose)
    assert rot < 1.0 and trans < 0.05


def test_sampling_gives_up_after_max_tries_on_an_empty_plane(api):
    """Hypotheses assigned to an expert whose plane is all zeros (train_esac.py:121 leaves inactive experts at zero) can
    never pass the 4-point gate: the loop must stop at MAX_SAMPLING_TRIES with the last try's state (esac_util.h:154)."""
    sc = make_scene(E=2, H=30, W=40, M=8, sub=8, seed=15)
    sc.coords[:] = 0.0
    api.set_option("max_tries", 3000)
    try:
        api.set_seed(1)
        out = np.zeros((4, 4), np.float32)
        api.forward(sc.coords, sc.assign, out, *sc.params)
        hy = api.last_hypotheses()
    finally:
        api.set_option("max_tries", 1000000)
    assert hy["tries"].tolist() == [3000] * 8
    assert np.all(hy["poses"] == 0)  # safeSolvePnP's failure state


# ---- every refinement walk against the cv2 oracle -------------------------------------------------------------------
# refine.cu has four ways to walk a CTA's share of `words` = ceil(N / 32) mask words, chosen per launch from the group size G:
# share <= kCacheWords (96) -> cells cached in shared memory, else read from global memory; and with refine_compact = 1 the
# LM evaluations walk a per-CTA inlier list (shared memory when cached, global scratch up to kMaxCompactWords = 2048),
# otherwise predicated passes over all cells.  At 60x80 (150 words) G = 1 is uncached and G >= 2 cached, so every walk runs.
REFINE_CACHE_WORDS, REFINE_COMPACT_WORDS = 96, 2048


def refine_walk(N, group, compact):
    words = (N + 31) // 32
    share = (words + group - 1) // group
    cached = share <= REFINE_CACHE_WORDS
    if compact and (cached or share <= REFINE_COMPACT_WORDS):
        return "shared-list" if cached else "global-list"
    return "cached-all-cells" if cached else "all-cells"


def perturbed_truth(sc, rng, M, rot=0.004, trans=0.02):
    """Ground truth with a small motion in the camera frame: every refinement round moves."""
    import cv2
    T = np.linalg.inv(sc.gt_pose.astype(np.float64))
    poses6 = np.zeros((M, 6))
    for h in range(M):
        dR, _ = cv2.Rodrigues(rng.normal(0, rot, 3))
        poses6[h, :3] = cv2.Rodrigues(dR @ T[:3, :3])[0].ravel()
        poses6[h, 3:] = dR @ T[:3, 3] + rng.normal(0, trans, 3)
    return poses6


WALK_SCENES = {
    "60x80-sub8": dict(E=2, H=60, W=80, M=12, sub=8, seed=6),
    "120x160-sub4": dict(E=2, H=120, W=160, M=14, sub=4, seed=12, noise=0.05, outlier_frac=0.3),
}


@pytest.fixture(scope="module", params=list(WALK_SCENES))
def walk_scene(request):
    """A scene, M >= 12 perturbed-truth poses on the ground-truth plane (so that jobs_hint >= 8) and the cv2 oracle's
    refineHyp of each, computed once."""
    kw = WALK_SCENES[request.param]
    sc = make_scene(**kw)
    M = kw["M"]
    assign = np.full(M, sc.gt_expert, np.int64)
    poses6 = perturbed_truth(sc, np.random.default_rng(kw["seed"]), M)
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


def test_every_refinement_walk_matches_oracle(api, walk_scene):
    """refine_group in {1, 2, auto, max} x refine_compact x refine_pretest x refine_jobs_per_group in {1, 3}: rounds and final
    inlier counts equal the oracle's and the poses are within 1e-3 deg / 1e-5 m of it; across variants rounds and inliers are
    identical and the poses equal up to the summation order (1e-9)."""
    import itertools
    name, sc, assign, poses6, ref = walk_scene
    N = sc.coords.shape[2] * sc.coords.shape[3]
    ctx = api.context()
    first, walks = None, set()
    try:
        for grp, compact, pretest, jpg in itertools.product((1, 2, 0, 1 << 20), (0, 1), (0, 1), (1, 3)):
            ctx.set_option("refine_group", grp)
            ctx.set_option("refine_compact", compact)
            ctx.set_option("refine_pretest", pretest)
            ctx.set_option("refine_jobs_per_group", jpg)
            got, rounds, inl = api.refine_poses(sc.coords, assign, poses6, sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy, sc.tau,
                                                sc.max_reproj, sc.sub)
            G = api.last_stats()["refine_group"]
            if grp in (1, 2):
                assert G == grp
            walks.add(refine_walk(N, G, compact))
            tag = (grp, G, compact, pretest, jpg)
            for h, (r, t, n_in, rr) in enumerate(ref):
                assert rounds[h] == rr and inl[h] == n_in, (tag, h, rounds[h], rr, inl[h], n_in)
                Ta, Tb = O.pose2trans(r, t), O.pose2trans(got[h, :3].reshape(3, 1), got[h, 3:].reshape(3, 1))
                rot, trans = pose_error(Tb, Ta)
                assert rot < ROT_TOL_DEG and trans < TRANS_TOL_M, (tag, h, rot, trans)
            if first is None:
                first = (got, rounds, inl)
            assert rounds.tolist() == first[1].tolist() and inl.tolist() == first[2].tolist(), tag
            assert np.abs(got - first[0]).max() < 1e-9, (tag, np.abs(got - first[0]).max())
    finally:
        ctx.set_option("refine_group", 0)
        ctx.set_option("refine_compact", 1)
        ctx.set_option("refine_pretest", 1)
        ctx.set_option("refine_jobs_per_group", 3)
    assert max(r[3] for r in ref) >= 1 and min(r[2] for r in ref) > 4       # every job was refined
    if name == "60x80-sub8":
        assert walks == {"shared-list", "global-list", "cached-all-cells", "all-cells"}, walks
