"""The sampling stage's float prefilter and early-exit verdict at every inlier threshold, on the host compile.  No GPU.

The prefilter (esac_p3p_fast.cuh) rejects a try only when every float P3P root misses the 4th point by more than its band,
and the exact verdict (hyp.cu) exits early when no unpolished candidate brings the 4th point within 1.25 tau + 1 px.  Both
bands depend on tau, while the float error they must cover is in pixels.  Held here at tau from 0.05 to 200 px, on random
draws of true and wrong experts of make_scene's maps (noise 5e-4 to 5e-2, room and world-offset outdoor scenes,
millimetre units, a shifted grid: >= 1e5 tries per tau) and on the crafted ill-conditioned sets of tests/minimal_sets.py:

  accept => may_pass    (esacb200_host_tries_hint: a try the exact path accepts is never thrown away), and the hint at
                        its largest fraction (1.99 tau) implies may_pass;
  early exit = full     (esacb200_host_try_verdict against esacb200_host_try's exact verdict).

A try the prefilter drops although the reference accepts it makes the device keep a later try than the reference."""
import ctypes as C

import numpy as np
import pytest

import minimal_sets as MS
from esac_b200.synth import make_scene

TAUS = (0.05, 0.1, 0.2, 0.3, 0.5, 0.6, 0.75, 1.0, 2.0, 5.0, 10.0, 25.0, 50.0, 100.0, 200.0)
HINT = 1.99           # the largest sample_hint the context accepts
N_DRAWS = 10000       # per scene and expert: 6 scenes x 2 experts ~ 1.2e5 tries per tau
N_VERDICT = 300       # tries per scene, expert and tau whose early-exit verdict is compared (those the prefilter passes first)
SCENES = {
    "room-noise5e-4": dict(E=2, H=60, W=80, M=8, sub=8, seed=3, noise=5e-4, active_only=False),
    "room-noise2e-3": dict(E=2, H=60, W=80, M=8, sub=8, seed=2, noise=0.002, active_only=False),
    "room-noise5e-2-shift": dict(E=2, H=60, W=80, M=8, sub=8, seed=4, noise=0.05, shiftX=3, shiftY=-5, active_only=False),
    "outdoor-world700": dict(E=2, H=48, W=64, M=8, sub=8, seed=5, noise=0.01, outdoor=True, world_offset=700.0,
                             active_only=False),
    "room-millimetres": dict(E=2, H=30, W=40, M=8, sub=8, seed=6, noise=0.002, unit_scale=1000.0, active_only=False),
    "room-noise1e-2-sub4": dict(E=2, H=60, W=80, M=8, sub=4, seed=7, noise=0.01, active_only=False),
}


def draws(sc, e, n, rng):
    """n random tries of 4 distinct cells on expert e's map, at the pixel centres of the (shifted) sampling grid:
    obj [n, 4, 3], img [n, 4, 2] (tests/test_host_sample_hint.py's draws, plus the shift)."""
    _, _, H, W = sc.coords.shape
    xs = rng.integers(0, W - 1, (n, 4))
    ys = rng.integers(0, H - 1, (n, 4))
    key = ys * W + xs
    distinct = np.array([len(set(k)) == 4 for k in key])
    xs, ys = xs[distinct], ys[distinct]
    obj = sc.coords[e][:, ys, xs].transpose(1, 2, 0)
    img = np.stack([xs * sc.sub + sc.sub // 2 - sc.shiftX, ys * sc.sub + sc.sub // 2 - sc.shiftY], -1)
    return obj, img


def tries(lib, obj, img, f, ppx, ppy, tau, hint=HINT):
    """(may_pass, hint, accept) of n tries as prefilter_kernel and the exact path see them."""
    n = len(obj)
    obj = np.ascontiguousarray(obj, np.float32)
    img = np.ascontiguousarray(img, np.float32)
    mp, hi, ac = (np.zeros(n, np.int32) for _ in range(3))
    lib.esacb200_host_tries_hint(n, obj.ctypes.data, img.ctypes.data, f, ppx, ppy, tau, hint, mp.ctypes.data, hi.ctypes.data,
                                 ac.ctypes.data)
    return mp.astype(bool), hi.astype(bool), ac.astype(bool)


def verdicts(lib, obj, img, f, ppx, ppy, tau):
    """(full exact verdict, early-exit verdict) of each try."""
    full, early = [], []
    mp, ac, ev = C.c_int(), C.c_int(), C.c_int()
    for o, i in zip(obj, img):
        o = np.ascontiguousarray(o, np.float32)
        i = np.ascontiguousarray(i, np.float32)
        lib.esacb200_host_try(o.ctypes.data, i.ctypes.data, f, ppx, ppy, tau, 2.0, C.byref(mp), C.byref(ac))
        lib.esacb200_host_try_verdict(o.ctypes.data, i.ctypes.data, f, ppx, ppy, tau, C.byref(ev), None)
        full.append(bool(ac.value))
        early.append(bool(ev.value))
    return np.array(full), np.array(early)


@pytest.fixture(scope="module")
def drawn():
    """Per scene: (scene, [(expert kind, obj, img)]), drawn once."""
    out = {}
    for k, (name, kw) in enumerate(SCENES.items()):
        sc = make_scene(**kw)
        rng = np.random.default_rng(100 + k)
        out[name] = (sc, [(which, *draws(sc, sc.gt_expert if which == "gt" else 1 - sc.gt_expert, N_DRAWS, rng))
                          for which in ("gt", "other")])
    return out


@pytest.mark.parametrize("tau", TAUS)
def test_random_draws_never_drop_an_accepted_try(lib, drawn, tau):
    n = n_acc = n_may = n_cmp = 0
    for name, (sc, sets) in drawn.items():
        for which, obj, img in sets:
            mp, hi, ac = tries(lib, obj, img, sc.f, sc.ppx, sc.ppy, tau)
            bad = np.flatnonzero(ac & ~mp)
            assert bad.size == 0, (name, which, tau, f"{bad.size} accepted tries rejected by the prefilter", bad[:8])
            assert not (hi & ~mp).any(), (name, which, tau, np.flatnonzero(hi & ~mp)[:8])
            # the verdict path on the tries the device would judge: those the prefilter lets through
            sel = np.flatnonzero(mp)[:N_VERDICT]
            full, early = verdicts(lib, obj[sel], img[sel], sc.f, sc.ppx, sc.ppy, tau)
            assert np.array_equal(full, ac[sel])
            diff = sel[full != early]
            assert diff.size == 0, (name, which, tau, "early-exit verdict differs from the full verdict", diff[:8])
            n += len(obj)
            n_acc += int(ac.sum())
            n_may += int(mp.sum())
            n_cmp += sel.size
    print(f"tau {tau:g}: {n} tries, {n_acc} accepted, {n_may} sent to the exact path, {n_cmp} verdicts compared")
    assert n >= 100000
    assert n_acc > 0 and n_may < n                  # both sides of the prefilter were exercised


@pytest.mark.parametrize("tau", TAUS)
def test_crafted_sets_never_drop_an_accepted_try(lib, tau):
    """Each family of tests/minimal_sets.py with its 4th point spread over [0, 1.2 tau) of the true pose, and its scaled and
    offset variants."""
    n_acc = 0
    for family in MS.FAMILIES:
        base = MS.generate(family, 40, seed=11, tau=tau)
        ts = base + MS.variants(base)
        obj = np.stack([t.obj for t in ts])
        img = np.stack([t.img() for t in ts])
        mp, hi, ac = tries(lib, obj, img, 525.0, MS.PPX, MS.PPY, tau)
        bad = np.flatnonzero(ac & ~mp)
        assert bad.size == 0, (family, tau, f"{bad.size} accepted tries rejected by the prefilter",
                               [ts[i].params for i in bad[:4]])
        assert not (hi & ~mp).any(), (family, tau)
        sel = np.flatnonzero(mp)[:N_VERDICT]
        full, early = verdicts(lib, obj[sel], img[sel], 525.0, MS.PPX, MS.PPY, tau)
        assert np.array_equal(full, ac[sel])
        diff = sel[full != early]
        assert diff.size == 0, (family, tau, "early-exit verdict differs", [ts[i].params for i in diff[:4]])
        n_acc += int(ac.sum())
    assert n_acc > 0


# ---- accepted tries at sub-pixel tau ---------------------------------------------------------------------------------
# Random draws rarely pass the gate below a pixel (78 of ~1.2e5 at tau = 0.05 above), so accept => may_pass is also held
# on low-noise true-expert draws, where thousands of tries are accepted at every sub-pixel tau.
SUBPX_TAUS = (0.05, 0.1, 0.2, 0.3, 0.5, 0.6, 0.75, 1.0)
SUBPX_SCENES = {
    "room-noise2e-3": (dict(E=2, H=60, W=80, M=8, sub=8, seed=2, noise=0.002, active_only=False), 2),
    "room-noise5e-4": (dict(E=2, H=60, W=80, M=8, sub=8, seed=3, noise=5e-4, active_only=False), 3),
    "outdoor-world700-noise1e-3": (dict(E=2, H=60, W=80, M=8, sub=8, seed=5, noise=0.001, outdoor=True, world_offset=700.0,
                                        active_only=False), 5),
    "room-millimetres-noise5e-4": (dict(E=2, H=60, W=80, M=8, sub=8, seed=6, noise=5e-4, unit_scale=1000.0,
                                        active_only=False), 6),
}


@pytest.fixture(scope="module")
def subpx_drawn():
    out = {}
    for name, (kw, seed) in SUBPX_SCENES.items():
        sc = make_scene(**kw)
        out[name] = (sc, *draws(sc, sc.gt_expert, 60000, np.random.default_rng(seed)))
    return out


@pytest.mark.parametrize("tau", SUBPX_TAUS)
def test_accepted_subpixel_tries_are_never_dropped(lib, subpx_drawn, tau):
    n_acc = 0
    for name, (sc, obj, img) in subpx_drawn.items():
        mp, hi, ac = tries(lib, obj, img, sc.f, sc.ppx, sc.ppy, tau)
        bad = np.flatnonzero(ac & ~mp)
        assert bad.size == 0, (name, tau, f"{bad.size} of {int(ac.sum())} accepted tries rejected by the prefilter", bad[:8])
        assert not (hi & ~mp).any(), (name, tau)
        n_acc += int(ac.sum())
    print(f"tau {tau:g}: {n_acc} accepted tries")
    assert n_acc >= 1000


# ---- the counterexample: a sub-pixel tau that a band of 2 tau alone could not cover ------------------------------------
COUNTER_SCENE = dict(E=2, H=60, W=80, M=8, sub=8, seed=2, noise=0.002, active_only=False)
COUNTER_TRY = 30541
COUNTER_IMG = [[596, 140], [124, 244], [36, 268], [20, 220]]


def counterexample():
    """Try 30541 of 40000 true-expert draws (tests/test_host_sample_hint.py's _draws, rng 2) on COUNTER_SCENE: (scene, obj
    [4, 3], img [4, 2], its four cells [4, 2] as (x, y))."""
    from test_host_sample_hint import _draws
    sc = make_scene(**COUNTER_SCENE)
    obj, img = _draws(sc, sc.gt_expert, 40000, np.random.default_rng(2))
    obj, img = obj[COUNTER_TRY], img[COUNTER_TRY]
    assert img.tolist() == COUNTER_IMG
    return sc, obj, img, (img - sc.sub // 2) // sc.sub


@pytest.mark.parametrize("tau", [0.5, 0.6])
def test_counterexample_at_subpixel_tau_is_not_dropped(lib, tau):
    """The exact pose puts the 4th point 0.4537 px off, so the exact path accepts at tau = 0.5 and 0.6; the float 4th point
    is over 0.7 px further off, outside a band of 2 tau (1.0 / 1.2 px)."""
    sc, obj, img, _ = counterexample()
    mp, hi, ac = tries(lib, obj[None], img[None], sc.f, sc.ppx, sc.ppy, tau)
    assert ac[0], "the exact path accepts the counterexample"
    assert mp[0], "the prefilter dropped a try the exact path accepts"
    pose = np.zeros(6)
    gate = C.c_int()
    o = np.ascontiguousarray(obj, np.float32)
    i = np.ascontiguousarray(img, np.float32)
    assert lib.esacb200_host_p3p_pose(o.ctypes.data, i.ctypes.data, sc.f, sc.ppx, sc.ppy, tau, pose.ctypes.data, C.byref(gate))
    import cv2
    R, _ = cv2.Rodrigues(pose[:3])
    X = R @ obj[3].astype(np.float64) + pose[3:]
    err = np.hypot(sc.f * X[0] / X[2] + sc.ppx - img[3, 0], sc.f * X[1] / X[2] + sc.ppy - img[3, 1])
    assert abs(err - 0.4537) < 1e-3, err
