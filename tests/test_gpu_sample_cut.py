"""The prefilter's window cut (option sample_hint) against the cv2 oracle's first accepted try (run with `-m gpu` on an H100).

prefilter_kernel raises a hint on a surviving try whose 4th point the float path puts within sample_hint * tau; the later
tries of that hypothesis' window are then not prefiltered, and advance_wave counts the hypothesis as resolved only when a
try up to the hinted one was accepted -- else the next wave resumes right after it.  Every try below the result is still
judged, so the kept try, its cells and its pose may not depend on the threshold.  Each test holds tries and cells exactly,
poses to 1e-8, to oracle.esac_oracle.sample_hypotheses and the poses bitwise to the same scene's default run, and shows
from Context.sample_profile() that the cut was (or was not) taken: tries_cut counts the tries the prefilter skipped,
hints_rejected the hinted tries the exact verdict rejected."""
import numpy as np
import pytest

from esac_b200.synth import make_scene
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-8
HINT_DEFAULT = 0.95        # capi_internal.h, struct Options::sample_hint
# the library's defaults (capi_internal.h, struct Options) of every option this module sets
LIBRARY_DEFAULTS = {"max_tries": 1000000, "sample_prefilter": 1, "sample_span0": 256, "sample_groups": 2, "upload_split": 1,
                    "sample_hint": HINT_DEFAULT, "fixed_seed": 0}


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    return api


def _restore(api):
    ctx = api.context()
    ctx.inject_cells(None)
    for k, v in LIBRARY_DEFAULTS.items():
        ctx.set_option(k, v)


@pytest.fixture(autouse=True)
def library_defaults(api):
    try:
        yield
    finally:
        _restore(api)


def _sample(api, sc, seed, inject=None, **opts):
    """One esac.forward under the options `opts` (fixed seed): (hypotheses, sample profile)."""
    ctx = api.context()
    try:
        ctx.set_option("fixed_seed", 1)
        for k, v in opts.items():
            ctx.set_option(k, v)
        api.set_seed(seed)
        if inject is not None:
            api.inject_cells(inject)
        out = np.zeros((4, 4), np.float32)
        api.forward(sc.coords, sc.assign, out, *sc.params)
        return api.last_hypotheses(), ctx.sample_profile()
    finally:
        _restore(api)


class Ref:
    def __init__(self, hyps):
        self.tries = np.array([h.tries for h in hyps], np.int32)
        self.cells = np.array([[list(c) for c in h.cells] for h in hyps], np.int32)
        self.poses = np.array([np.concatenate([h.rvec.ravel(), h.tvec.ravel()]) for h in hyps])


def _oracle(sc, seed, max_tries=O.MAX_SAMPLING_TRIES, injected=None):
    K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
    H, W = sc.coords.shape[2:]
    sampling = O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY)
    return Ref(O.sample_hypotheses(sc.coords, sc.assign, sampling, K, max_tries, sc.tau, seed, injected))


def _assert_matches(hy, ref, base=None):
    tries, cells, poses = hy["tries"], hy["cells"], hy["poses"]
    bad = np.flatnonzero(tries != ref.tries)
    assert bad.size == 0, ("tries", bad[:8], tries[bad[:8]], ref.tries[bad[:8]])
    bad = np.flatnonzero((cells != ref.cells).any(axis=(1, 2)))
    assert bad.size == 0, ("cells", bad[:8])
    err = np.abs(poses - ref.poses).max(axis=1)
    assert err.max() < POSE_TOL, ("poses", np.flatnonzero(err >= POSE_TOL)[:8], err.max())
    if base is not None:
        for k in ("tries", "cells", "poses"):
            assert np.array_equal(hy[k], base[k]), (k, "differs bitwise from the default run")


class Case:
    def __init__(self, api, sc, seed, max_tries=O.MAX_SAMPLING_TRIES, inject=None, **default_opts):
        self.sc, self.seed, self.max_tries, self.inject = sc, seed, max_tries, inject
        self.ref = _oracle(sc, seed, max_tries, inject)
        self.base, self.base_prof = _sample(api, sc, seed, inject=inject, max_tries=max_tries, **default_opts)
        print("default", self.base_prof)
        _assert_matches(self.base, self.ref)

    def run(self, api, **opts):
        hy, prof = _sample(api, self.sc, self.seed, inject=self.inject, max_tries=self.max_tries, **opts)
        print(opts, prof)
        _assert_matches(hy, self.ref, self.base)
        return hy, prof


@pytest.fixture(scope="module")
def scene_e2(api):
    return Case(api, make_scene(E=2, H=30, W=40, M=64, sub=8, seed=31), 501)


@pytest.fixture(scope="module")
def scene_e4(api):
    return Case(api, make_scene(E=4, H=30, W=40, M=64, sub=8, seed=32, shiftX=3, shiftY=-4), 502)


@pytest.fixture(scope="module")
def scene_lanes(api):
    """N = 65536 cells, M = 512: the lane count follows sample_groups (max_tries = 2000 bounds the oracle's work)."""
    sc = make_scene(E=6, H=256, W=256, M=512, sub=8, seed=33, gt_mass=0.95)
    case = Case(api, sc, 505, max_tries=2000, upload_split=0)
    assert np.isfinite(case.ref.poses).all()
    return case


@pytest.fixture(scope="module")
def scene_injected(api):
    """scene_e2's maps with injected random minimal sets (4 distinct cells each), 8192 per hypothesis."""
    sc = make_scene(E=2, H=30, W=40, M=64, sub=8, seed=36)
    T = 8192
    rng = np.random.default_rng(9)
    _, _, H, W = sc.coords.shape
    n = (W - 1) * (H - 1)
    k = rng.integers(0, n, (len(sc.assign), T, 4))
    while True:   # redraw the sets with a repeated cell
        s = np.sort(k, axis=-1)
        dup = (np.diff(s, axis=-1) == 0).any(axis=-1)
        if not dup.any():
            break
        k[dup] = rng.integers(0, n, (int(dup.sum()), 4))
    cells = np.stack([k % (W - 1), k // (W - 1)], -1).astype(np.int32)
    return Case(api, sc, 0, inject=cells)


@pytest.mark.parametrize("scene", ["scene_e2", "scene_e4"])
def test_hint_off_and_default_match_oracle(api, request, scene):
    case = request.getfixturevalue(scene)
    _, off = case.run(api, sample_hint=0)
    assert off["tries_cut"] == 0 and off["hints_rejected"] == 0
    _, nopf = case.run(api, sample_prefilter=0)       # no prefilter, no hint
    assert nopf["tries_cut"] == 0 and nopf["hints_rejected"] == 0
    assert nopf["tries_prefiltered"] == nopf["survivors_judged"]


@pytest.mark.parametrize("scene", ["scene_e2", "scene_e4"])
def test_false_hints_resume_after_the_hinted_try(api, request, scene):
    """At 1.9 tau most hints on the true expert are false: the hinted try is rejected, the window was cut after it, and
    the next wave (or the tail) resumes there.  A first window of 65536 tries makes the cut reachable on these maps."""
    case = request.getfixturevalue(scene)
    _, prof = case.run(api, sample_hint=1.9)
    assert prof["hints_rejected"] > 0
    _, prof = case.run(api, sample_hint=1.9, sample_span0=65536)
    assert prof["hints_rejected"] > 0 and prof["tries_cut"] > 0


@pytest.mark.parametrize("hint", [HINT_DEFAULT, 1.9])
def test_cut_with_survivor_overflow(api, scene_e2, hint):
    """A first window of 65536 tries: without the cut the true expert's survivors overflow the list; with it, hints cut
    the windows in the same wave as the list may still overflow, and the resume point is the lower of the two."""
    _, prof = scene_e2.run(api, sample_hint=hint, sample_span0=65536)
    assert prof["tries_cut"] > 0
    _, off = scene_e2.run(api, sample_hint=0, sample_span0=65536)
    assert off["tries_cut"] == 0


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_cut_on_lanes(api, scene_lanes, groups):
    for hint in (HINT_DEFAULT, 1.9):
        _, prof = scene_lanes.run(api, sample_groups=groups, upload_split=0, sample_hint=hint)
        assert prof["lanes"] == groups


@pytest.mark.parametrize("hint", [0, HINT_DEFAULT, 1.9])
def test_cut_on_injected_cells(api, scene_injected, hint):
    _, prof = scene_injected.run(api, sample_hint=hint, sample_span0=8192)
    assert (prof["tries_cut"] > 0) == (hint > 0)


def test_bench_scene_cut_changes_nothing(api):
    """A bench-shaped scene (7 experts x 256 hypotheses, 480x640, subSampling 1): the default cuts windows, and every
    hypothesis' tries, cells and pose are bitwise those of sample_hint = 0 (no oracle: ~1e3 tries per wrong-expert
    hypothesis on 1792 hypotheses is beyond it)."""
    sc = make_scene(E=7, H=480, W=640, M=256, sub=1, seed=100, per_expert=True, active_only=False)
    on, p_on = _sample(api, sc, 7)
    off, p_off = _sample(api, sc, 7, sample_hint=0)
    print("default", p_on, "off", p_off)
    for k in ("tries", "cells", "poses"):
        assert np.array_equal(on[k], off[k]), k
    assert p_on["tries_cut"] > 0 and p_off["tries_cut"] == 0
    assert p_on["tries_prefiltered"] - p_on["tries_cut"] < p_off["tries_prefiltered"]
