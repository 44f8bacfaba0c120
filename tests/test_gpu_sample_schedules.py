"""Every sampling schedule against the cv2 oracle's first accepted try (run with `-m gpu` on an H100).

The sampling stage (esac_b200/csrc/hyp.cu) evaluates tries in bulk -- waves of prefilter_kernel -> exact_kernel whose
windows advance_wave picks on the device, then tail_kernel, then emit_kernel, on one to four lanes -- but must keep, for
every hypothesis, the lowest try that passes the 4-point gate: the try the reference's sequential loop stops at
(esac_util.h:129-225), with that try's cells and pose; an exhausted hypothesis keeps the state of try limit - 1.  How
many lanes and waves run, how wide the windows are and whether the survivor list or the staging area overflows may not
change the result.  Each test below forces one schedule through the context's options, shows from
Context.sample_profile() that the schedule was taken, and holds tries and cells exactly, poses to 1e-8, to
oracle.esac_oracle.sample_hypotheses (cv2 solvePnP(P3P) in float64 and the reference's float-rounded gate), and the
poses bitwise to the same scene's default schedule."""
import contextlib

import numpy as np
import pytest

from esac_b200.synth import Scene, make_scene
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-8            # test_gpu_forward.py::test_sampling_matches_oracle_stream
SAMPLE_CAP = 1 << 19       # capi_pipeline.cu kSampleCap: survivors per lane and wave
SAMPLE_CAP_ACC = 1 << 15   # capi_pipeline.cu kSampleCapAcc: staged accepts per lane and call
FIXED_SEED = 1             # every call of this module draws from set_seed's seed itself
# the library's defaults (capi_internal.h, struct Options) of every option this module sets
LIBRARY_DEFAULTS = {"max_tries": 1000000, "sample_prefilter": 1, "sample_span0": 256, "sample_window": 1.25,
                    "sample_waves": 6, "sample_tail_boost": 1, "sample_groups": 2, "sample_trace": 0, "upload_split": 1,
                    "hyp_offset": 0, "hyp_stride": 1, "fixed_seed": 0}


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    return api


def _restore(api):
    """The context's options are global to the process: put back what a fresh context has."""
    ctx = api.context()
    ctx.inject_cells(None)
    for k, v in LIBRARY_DEFAULTS.items():
        ctx.set_option(k, v)


@contextlib.contextmanager
def _schedule(api, **opts):
    ctx = api.context()
    try:
        ctx.set_option("fixed_seed", FIXED_SEED)
        for k, v in opts.items():
            ctx.set_option(k, v)
        yield ctx
    finally:
        _restore(api)


@pytest.fixture(autouse=True)
def library_defaults(api):
    """Whatever a test sets, and however it ends, the next test (in this module or another) starts from the defaults."""
    try:
        yield
    finally:
        _restore(api)


def _sample(api, sc, seed, coords=None, inject=None, **opts):
    """One esac.forward under the options `opts`: (hypotheses, sample profile, pose, expert)."""
    with _schedule(api, **opts) as ctx:
        api.set_seed(seed)
        if inject is not None:
            api.inject_cells(inject)
        out = np.zeros((4, 4), np.float32)
        e = api.forward(sc.coords if coords is None else coords, sc.assign, out, *sc.params)
        return api.last_hypotheses(), ctx.sample_profile(), out, e


class Ref:
    """The oracle's hypotheses as arrays."""

    def __init__(self, hyps):
        self.tries = np.array([h.tries for h in hyps], np.int32)
        self.cells = np.array([[list(c) for c in h.cells] for h in hyps], np.int32)
        self.poses = np.array([np.concatenate([h.rvec.ravel(), h.tvec.ravel()]) for h in hyps])


def _oracle(sc, seed, max_tries=O.MAX_SAMPLING_TRIES, injected=None):
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    H, W = sc.coords.shape[2:]
    sampling = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY)
    return Ref(O.sample_hypotheses(sc.coords, sc.assign, sampling, K, max_tries, sc.tau, seed, injected))


def _assert_matches(hy, ref, base=None, rows=slice(None)):
    """tries and cells exactly, poses to POSE_TOL of the oracle and bitwise to `base` (the default schedule's run)."""
    tries, cells, poses = hy["tries"], hy["cells"], hy["poses"]
    bad = np.flatnonzero(tries != ref.tries[rows])
    assert bad.size == 0, ("tries", bad[:8], tries[bad[:8]], ref.tries[rows][bad[:8]])
    bad = np.flatnonzero((cells != ref.cells[rows]).any(axis=(1, 2)))
    assert bad.size == 0, ("cells", bad[:8])
    err = np.abs(poses - ref.poses[rows]).max(axis=1)
    assert err.max() < POSE_TOL, ("poses", np.flatnonzero(err >= POSE_TOL)[:8], err.max())
    if base is not None:
        bad = np.flatnonzero((poses != base["poses"][rows]).any(axis=1))
        assert bad.size == 0, ("poses differ bitwise from the default schedule", bad[:8])


class Case:
    def __init__(self, api, sc, seed, max_tries=O.MAX_SAMPLING_TRIES, **default_opts):
        self.sc, self.seed, self.max_tries = sc, seed, max_tries
        self.ref = _oracle(sc, seed, max_tries)
        self.base, self.base_prof, _, _ = _sample(api, sc, seed, max_tries=max_tries, **default_opts)
        _assert_matches(self.base, self.ref)

    def run(self, api, **opts):
        hy, prof, _, _ = _sample(api, self.sc, self.seed, max_tries=self.max_tries, **opts)
        print(opts, prof)
        _assert_matches(hy, self.ref, self.base)
        return hy, prof


# ---- scenes: the oracle runs once per scene; wrong-expert hypotheses need ~1e3 tries on the 30x40 maps ----------------
@pytest.fixture(scope="module")
def scene_e2(api):
    return Case(api, make_scene(E=2, H=30, W=40, M=64, sub=8, seed=31), 501)


@pytest.fixture(scope="module")
def scene_e4(api):
    return Case(api, make_scene(E=4, H=30, W=40, M=64, sub=8, seed=32, shiftX=3, shiftY=-4), 502)


@pytest.fixture(scope="module")
def scene_lanes(api):
    """N = 65536 cells and M = 512: the map on which the lane count follows sample_groups.  Wrong experts need ~5e4 tries
    on this map, so max_tries = 2000 (not a multiple of 256) keeps the oracle at ~5e4 tries in all and ~20 hypotheses end
    exhausted; the host maps (4.5 MB) are above the split-upload threshold, which upload_split = 0 turns off for the
    default run.  On a few last tries of an exhausted hypothesis OpenCV 4.13's solvePnP reports success with a NaN
    translation, which no tolerance can compare; the stream seed is one on which no hypothesis ends on such a try."""
    sc = make_scene(E=6, H=256, W=256, M=512, sub=8, seed=33, gt_mass=0.95)
    case = Case(api, sc, 505, max_tries=2000, upload_split=0)
    assert (case.ref.tries == 2000).sum() >= 16 and np.isfinite(case.ref.poses).all()
    return case


@pytest.fixture(scope="module")
def scene_stage(api):
    """Noise-free, outlier-free single expert: nearly every try passes the gate."""
    return Case(api, make_scene(E=1, H=60, W=80, M=64, sub=8, seed=34, outlier_frac=0.0, noise=0.0), 504)


# ---- 1. schedule matrix on the counter stream -------------------------------------------------------------------------
SCHEDULES = {
    "waves0": dict(sample_waves=0),
    "waves1": dict(sample_waves=1),
    "waves2_noprefilter": dict(sample_waves=2, sample_prefilter=0),
    "waves64_window0.05": dict(sample_waves=64, sample_window=0.05),   # the smallest windows: 256 tries
    "span1280": dict(sample_span0=1280),
    "span1280_window0.05_noprefilter": dict(sample_span0=1280, sample_window=0.05, sample_prefilter=0),
    "span65536": dict(sample_span0=65536),    # survivors of the correct expert's tries overflow the list
    "window8_boost16": dict(sample_window=8, sample_tail_boost=16),
    "window0.05_boost16_waves2": dict(sample_window=0.05, sample_tail_boost=16, sample_waves=2),
    "noprefilter": dict(sample_prefilter=0),
}


@pytest.mark.parametrize("name", list(SCHEDULES))
@pytest.mark.parametrize("scene", ["scene_e2", "scene_e4"])
def test_schedule_matches_oracle(api, request, scene, name):
    case = request.getfixturevalue(scene)
    opts = SCHEDULES[name]
    _, prof = case.run(api, **opts)
    M = len(case.sc.assign)
    waves = opts.get("sample_waves", 6)
    span0 = opts.get("sample_span0", 256)
    assert prof["lanes"] == 1
    assert prof["waves"] <= waves
    if prof["left_to_tail"] > 0:          # something reached the tail: every wave had work
        assert prof["waves"] == waves
    if waves > 0:                         # the first wave judged span0 tries of every hypothesis
        assert prof["tries_prefiltered"] >= M * span0
    if waves > 0 and not opts.get("sample_prefilter", 1) and span0 * M <= SAMPLE_CAP:
        assert prof["tries_prefiltered"] == prof["survivors_judged"]
    elif waves > 0:
        assert prof["survivors_judged"] < prof["tries_prefiltered"]
    if name == "waves0":
        assert prof["left_to_tail"] == M and prof["waves"] == 0 and prof["tries_prefiltered"] == 0
    if name in ("waves64_window0.05", "span65536"):   # the waves left nothing to the tail
        assert prof["left_to_tail"] == 0
    if name in ("waves1", "window0.05_boost16_waves2"):
        assert prof["left_to_tail"] > 0


# ---- 2. lanes -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_lanes_match_oracle(api, scene_lanes, groups):
    """512 hypotheses dealt to 1-4 lanes by index modulo the lane count (three lanes: 171, 171 and 170)."""
    _, prof = scene_lanes.run(api, sample_groups=groups, upload_split=0)
    assert prof["lanes"] == groups


def test_split_upload_lanes_by_expert_match_oracle(api, scene_lanes):
    """Pinned host maps above 4 MB are uploaded in two halves and the lanes are dealt by expert (lane 0 samples the first
    half's experts while the second half is on the wire).  Two lanes where sample_groups = 4 would otherwise run four
    shows the split was taken."""
    import torch
    sc = scene_lanes.sc
    assert sc.coords.nbytes >= 4 << 20
    pinned = torch.from_numpy(sc.coords).pin_memory()
    hy, prof, _, _ = _sample(api, sc, scene_lanes.seed, coords=pinned, max_tries=2000, sample_groups=4, upload_split=1)
    print(prof)
    assert prof["lanes"] == 2
    _assert_matches(hy, scene_lanes.ref, scene_lanes.base)


# ---- 3. / 4. window edges and exhausted hypotheses by injection -----------------------------------------------------------
INJ_T = 3000
EDGES = [0, 1, 127, 128, 255, 256, 257, 511, 512, 1023, 1024, 1025, 2047, 2048, 2499, 2999]
# exhausted hypotheses: the kind of their tries 2499 and 2999 (the last try at max_tries = 2500 and at T = 3000)
EXHAUSTED = ["solved", "solved", "unsolvable", "unsolvable"]


def _scene_errors(sc):
    """Reprojection error (px) of every cell of expert 0 under the ground-truth pose, [H, W]."""
    T = np.linalg.inv(sc.gt_pose.astype(np.float64))  # camera -> world into world -> camera
    _, _, H, W = sc.coords.shape
    X = sc.coords[0].reshape(3, -1).astype(np.float64)
    c = T[:3, :3] @ X + T[:3, 3:]
    s = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY).reshape(-1, 2)
    u = sc.f * c[0] / c[2] + sc.ppx
    v = sc.f * c[1] / c[2] + sc.ppy
    err = np.hypot(u - s[:, 0], v - s[:, 1])
    err[c[2] <= 0] = np.inf
    return err.reshape(H, W)


def _classify(sc, sets):
    """Oracle verdict of each candidate minimal set [n, 4, 2]: each is tried twice as its own hypothesis, so tries == 1
    means it passes the gate; otherwise the pose left is that of the set's own solve: zeros where safeSolvePnP failed,
    finite where it solved (OpenCV 4.13 also reports success with a NaN translation on some degenerate sets, e.g. a
    repeated cell: those are left out)."""
    n = len(sets)
    probe = Scene(sc.coords, np.zeros(n, np.int64), sc.gt_pose, 0, sc.f, sc.ppx, sc.ppy, sc.sub)
    ref = _oracle(probe, 0, 2, np.repeat(np.asarray(sets, np.int32)[:, None], 2, axis=1))
    accept = ref.tries == 1
    finite = np.isfinite(ref.poses).all(axis=1)
    zero = (ref.poses == 0).all(axis=1)
    return accept, finite & ~zero, zero


def _build_injection():
    """Minimal sets built so that each hypothesis' first accepting try sits on a window or chunk edge (EDGES: 256-try
    windows and prefilter passes, 128 = the split of a prefilter thread's two tries, 1024 = tail_kernel's chunks, 2499 /
    2999 = limit - 1), plus hypotheses that never accept.  Accepting sets are four well-spread inlier cells of a noise-free
    single-expert scene (one per quadrant); rejecting sets are four outlier cells, either solvable and gated out or with no
    P3P solution (safeSolvePnP fails, ~1% of them).  After the first accept, accepting and rejecting sets alternate at random, so a
    kernel that kept a later accept would show."""
    sc = make_scene(E=1, H=30, W=40, M=len(EDGES) + len(EXHAUSTED), sub=8, seed=35, outlier_frac=0.5, noise=0.0)
    _, _, H, W = sc.coords.shape
    err = _scene_errors(sc)
    rng = np.random.default_rng(7)
    inl = np.argwhere(err < 1.0)[:, ::-1]    # (x, y)
    outl = np.argwhere(err > 50.0)[:, ::-1]

    def quadrant_set():
        out = []
        for qx in (0, 1):
            for qy in (0, 1):
                m = ((inl[:, 0] >= W // 2) == qx) & ((inl[:, 1] >= H // 2) == qy)
                out.append(inl[m][rng.integers(m.sum())])
        return out

    acc_c = [quadrant_set() for _ in range(64)]
    rej_c = [outl[rng.choice(len(outl), 4, replace=False)] for _ in range(2000)]
    a_acc, _, _ = _classify(sc, acc_c)
    r_acc, r_sol, r_uns = _classify(sc, rej_c)
    acc = np.asarray(acc_c, np.int32)[a_acc]
    sol = np.asarray(rej_c, np.int32)[~r_acc & r_sol][:64]
    uns = np.asarray(rej_c, np.int32)[~r_acc & r_uns]
    assert len(acc) >= 48 and len(sol) == 64 and len(uns) >= 8, (len(acc), len(sol), len(uns))
    rej = np.concatenate([sol, uns])

    M = len(sc.assign)
    cells = rej[rng.integers(len(rej), size=(M, INJ_T))]
    for h, t in enumerate(EDGES):
        cells[h, t] = acc[rng.integers(len(acc))]
        later = np.arange(t + 1, INJ_T)
        hits = later[rng.random(later.size) < 0.5]
        cells[h, hits] = acc[rng.integers(len(acc), size=hits.size)]
    for k, kind in enumerate(EXHAUSTED):
        pool = sol if kind == "solved" else uns
        cells[len(EDGES) + k, [2499, 2999]] = pool[rng.integers(len(pool), size=2)]

    refs = {}
    for limit in (INJ_T, 2500):
        ref = _oracle(sc, 0, limit, cells)
        # the construction: the oracle stops exactly where intended
        want = [t + 1 if t < limit else limit for t in EDGES] + [limit] * len(EXHAUSTED)
        assert ref.tries.tolist() == want
        ex = ref.poses[len(EDGES):]
        assert [bool((p != 0).any()) for p in ex] == [k == "solved" for k in EXHAUSTED] and np.isfinite(ref.poses).all()
        refs[limit] = ref
    return sc, cells, refs


@pytest.fixture(scope="module")
def injected():
    return _build_injection()


INJ_SCHEDULES = {
    "default": dict(),
    "waves0": dict(sample_waves=0),
    "waves64_window0.05": dict(sample_waves=64, sample_window=0.05),
    "span1280": dict(sample_span0=1280),
    "window0.05": dict(sample_window=0.05),
    "noprefilter": dict(sample_prefilter=0),
}


@pytest.mark.parametrize("name", list(INJ_SCHEDULES))
@pytest.mark.parametrize("limit", [INJ_T, 2500], ids=["limit=T", "max_tries=2500"])
def test_first_accept_on_window_edges(api, injected, limit, name):
    """limit = T = 3000 (max_tries at its default), then max_tries = 2500 < T, which moves limit - 1 as well."""
    sc, cells, refs = injected
    opts = dict(INJ_SCHEDULES[name], max_tries=limit if limit < INJ_T else LIBRARY_DEFAULTS["max_tries"])
    base, _, _, _ = _sample(api, sc, 0, inject=cells, max_tries=opts["max_tries"])
    hy, prof, _, _ = _sample(api, sc, 0, inject=cells, **opts)
    print(name, limit, prof)
    _assert_matches(base, refs[limit])
    _assert_matches(hy, refs[limit], base)
    if name == "waves0":
        assert prof["left_to_tail"] == len(sc.assign)
    if name == "waves64_window0.05":      # windows of 256 tries up to the limit: more than the default six waves
        assert prof["waves"] > 6 and prof["left_to_tail"] == 0


@pytest.mark.parametrize("waves", [6, 0])
def test_exhausted_hypotheses_keep_the_last_try(api, injected, waves):
    """A hypothesis that never passes the gate keeps try limit - 1: its cells and, when that try solves but is gated out,
    its pose; zeros (safeSolvePnP's failure state) when it cannot be solved."""
    sc, cells, refs = injected
    ref = refs[INJ_T]
    hy, prof, _, _ = _sample(api, sc, 0, inject=cells, sample_waves=waves)
    ex = slice(len(EDGES), None)
    assert (hy["tries"][ex] == INJ_T).all()
    assert (hy["cells"][ex] == cells[ex, INJ_T - 1]).all()
    solved = np.array([k == "solved" for k in EXHAUSTED])
    assert (hy["poses"][ex][solved] != 0).all(axis=1).all()
    assert (hy["poses"][ex][~solved] == 0).all()
    _assert_matches(hy, ref)
    if waves == 0:
        assert prof["left_to_tail"] == len(sc.assign)


# ---- 5. / 6. overflows --------------------------------------------------------------------------------------------------
def test_survivor_list_overflow(api, scene_e2):
    """Prefilter off and a first window of 16384 tries: 64 x 16384 survivors, twice the list's capacity.  Where the list
    overflows is decided by the order in which CTAs append, which the test does not control, and that is intended: a
    hypothesis whose survivors did not fit resumes from its first lost try, an accept beyond that hole does not count
    yet, and the result must not depend on where the hole fell."""
    case = scene_e2
    M = len(case.sc.assign)
    _, prof = case.run(api, sample_prefilter=0, sample_span0=16384)
    assert prof["tries_prefiltered"] >= M * 16384 > SAMPLE_CAP
    assert prof["tries_prefiltered"] > prof["survivors_judged"]   # survivors were lost to the overflow ...
    # ... and every first accept lies inside the first window, so a second wave only had work because some hypothesis'
    # first accept lay beyond its hole
    assert case.ref.tries.max() <= 16384
    assert prof["waves"] >= 2


def test_staging_overflow(api, scene_stage):
    """A first window of 4096 tries on a map where nearly every try accepts: ~262k accepts against a staging area of
    32768, so the hypotheses whose accept came late lose their slot and emit_kernel solves their try again on the full
    P3P path.  Its pose must equal, bit for bit, the staged pose of the verdict path (a first window of 256 stages every
    accept)."""
    case = scene_stage
    _, prof = case.run(api, sample_span0=4096)
    assert prof["accepted_staged"] >= 4 * SAMPLE_CAP_ACC
    assert case.base_prof["accepted_staged"] <= SAMPLE_CAP_ACC


# ---- 7. trace -----------------------------------------------------------------------------------------------------------
def test_trace_stamps_only_the_first_32_waves(api, scene_e2):
    """The trace holds 32 waves per lane: with 40 waves on one lane, waves 32-39 run but are not stamped (before, they
    stamped lane 1's rows), and tracing does not change what is sampled."""
    case = scene_e2
    plain, prof, _, _ = _sample(api, case.sc, case.seed, sample_waves=40)
    with _schedule(api, sample_waves=40, sample_trace=1) as ctx:
        api.set_seed(case.seed)
        out = np.zeros((4, 4), np.float32)
        api.forward(case.sc.coords, case.sc.assign, out, *case.sc.params)
        traced, tr = api.last_hypotheses(), ctx.sample_trace()
    assert prof["lanes"] == 1
    assert (tr[0] >= 0).all()              # lane 0: waves 0-31, both kernels, start and end
    assert (tr[1:] == -1).all()            # nothing else ran
    for k in ("tries", "cells", "poses"):
        assert np.array_equal(traced[k], plain[k]), k
    _assert_matches(plain, case.ref, case.base)


# ---- 8. shard draws -----------------------------------------------------------------------------------------------------
def test_shard_draws_equal_the_rows_of_the_full_problem(api, scene_e2):
    """A shard draws the stream of the unsharded problem: hypothesis h of a shard is global hypothesis
    hyp_offset + h * hyp_stride, dealt round-robin (stride 2) or in contiguous halves (offset K)."""
    case = scene_e2
    full = case.base
    M = len(case.sc.assign)
    K = M // 2
    shards = [(slice(r, None, 2), dict(hyp_offset=r, hyp_stride=2)) for r in (0, 1)]
    shards += [(slice(r * K, (r + 1) * K), dict(hyp_offset=r * K)) for r in (0, 1)]
    for rows, opts in shards:
        sub = Scene(case.sc.coords, case.sc.assign[rows].copy(), case.sc.gt_pose, case.sc.gt_expert,
                                              case.sc.f, case.sc.ppx, case.sc.ppy, case.sc.sub)
        hy, _, _, _ = _sample(api, sub, case.seed, **opts)
        for k in ("tries", "cells", "poses"):
            assert np.array_equal(hy[k], full[k][rows]), (opts, k)
        _assert_matches(hy, case.ref, rows=rows)


# ---- 9. the stream-ordered path under forced schedules ---------------------------------------------------------------
ASYNC = {
    "waves0": ("scene_e2", dict(sample_waves=0)),
    "four_lanes": ("scene_lanes", dict(sample_groups=4, max_tries=2000)),
    "survivor_overflow": ("scene_e2", dict(sample_prefilter=0, sample_span0=16384)),
    "staging_overflow": ("scene_stage", dict(sample_span0=4096)),
}


@pytest.fixture
def own_context(api):
    """A context of its own for the test: the stream-ordered workspace of the shared one may be pinned by a graph that an
    earlier test captured at a smaller shape."""
    import torch
    dev = torch.cuda.current_device()
    saved = api._contexts.get(dev)
    ctx = api.Context(dev)
    api._contexts[dev] = ctx
    try:
        yield ctx
    finally:
        if saved is not None:
            api._contexts[dev] = saved
        else:
            api._contexts.pop(dev, None)
        ctx.close()


@pytest.mark.parametrize("name", list(ASYNC))
def test_forward_async_equals_eager_under_forced_schedule(api, request, name):
    """forward_async copies the context's options on every call, so its DEV kernels run the same schedule; its profile
    is not readable, so the eager run on the same inputs shows the path was reached."""
    import torch
    scene, opts = ASYNC[name]
    case = request.getfixturevalue(scene)
    request.getfixturevalue("own_context")
    sc = case.sc
    coords = torch.from_numpy(sc.coords).cuda()
    assign = torch.from_numpy(sc.assign).cuda()
    hy, prof, eager, e = _sample(api, sc, case.seed, coords=coords, **opts)
    print(name, prof)
    _assert_matches(hy, case.ref, case.base)
    if name == "waves0":
        assert prof["left_to_tail"] == len(sc.assign)
    elif name == "four_lanes":
        assert prof["lanes"] == 4
    elif name == "survivor_overflow":
        assert prof["tries_prefiltered"] > prof["survivors_judged"]
    else:
        assert prof["accepted_staged"] >= 4 * SAMPLE_CAP_ACC
    with _schedule(api, **opts):
        api.set_seed(case.seed)
        out = torch.zeros(4, 4, device="cuda")
        ex = torch.zeros((), dtype=torch.int64, device="cuda")
        st = torch.zeros((), dtype=torch.int32, device="cuda")
        api.forward_async(coords, assign, torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda"),
                          torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda"), sc.tau, sc.alpha, sc.beta, sc.max_reproj,
                          sc.sub, out, ex, st)
        torch.cuda.synchronize()
    assert int(st) == 0 and int(ex) == e
    np.testing.assert_array_equal(out.cpu().numpy(), eager)
