"""The prefilter's "near-certain" hint (option sample_hint), on the host compile of its code.  No GPU.

prefilter_kernel cuts a hypothesis' window at a hinted survivor: the later tries of the window are not prefiltered, and the
hypothesis resumes after the hinted try when the exact verdict rejects it.  That is only sound when a hinted try is one the
prefilter lets through (hint implies may-pass), which these tests hold on random draws of make_scene's maps (true and wrong
experts) and on the crafted ill-conditioned sets of tests/minimal_sets.py, at hint thresholds up to the option's 1.99."""
import numpy as np
import pytest

import minimal_sets as MS

HINTS = (0.5, 0.9, 1.5, 1.99)


def _tries(lib, obj, img, f, ppx, ppy, tau, hint):
    n = len(obj)
    obj = np.ascontiguousarray(obj, np.float32)
    img = np.ascontiguousarray(img, np.float32)
    mp, hi, ac = (np.zeros(n, np.int32) for _ in range(3))
    lib.esacb200_host_tries_hint(n, obj.ctypes.data, img.ctypes.data, f, ppx, ppy, tau, hint, mp.ctypes.data, hi.ctypes.data,
                                 ac.ctypes.data)
    return mp.astype(bool), hi.astype(bool), ac.astype(bool)


def _draws(sc, e, n, rng):
    """n random tries of 4 distinct cells on expert e's map: obj [n, 4, 3], img [n, 4, 2]."""
    _, _, H, W = sc.coords.shape
    xs = rng.integers(0, W - 1, (n, 4))
    ys = rng.integers(0, H - 1, (n, 4))
    key = ys * W + xs
    distinct = np.array([len(set(k)) == 4 for k in key])
    xs, ys = xs[distinct], ys[distinct]
    obj = sc.coords[e][:, ys, xs].transpose(1, 2, 0)
    img = np.stack([xs * sc.sub + sc.sub // 2, ys * sc.sub + sc.sub // 2], -1)
    return obj, img


@pytest.mark.parametrize("which", ["gt", "other"])
def test_hint_implies_may_pass_on_random_draws(lib, which):
    from esac_b200.synth import make_scene
    sc = make_scene(E=2, H=60, W=80, M=8, sub=8, seed=1, active_only=False)
    e = sc.gt_expert if which == "gt" else 1 - sc.gt_expert
    obj, img = _draws(sc, e, 20000, np.random.default_rng(11))
    for hint in HINTS:
        mp, hi, ac = _tries(lib, obj, img, sc.f, sc.ppx, sc.ppy, sc.tau, hint)
        assert not (hi & ~mp).any(), (hint, np.flatnonzero(hi & ~mp)[:8])
        assert not (ac & ~mp).any()
        if which == "gt":
            assert hi.sum() > 200                           # the hint was exercised ...
            if hint <= 0.9:                                 # ... and below tau it is nearly always right
                assert (ac & hi).sum() >= 0.95 * hi.sum(), (hint, (ac & hi).sum(), hi.sum())
    _, off, _ = _tries(lib, obj, img, sc.f, sc.ppx, sc.ppy, sc.tau, 0.0)
    assert not off.any()                                    # 0 = off


@pytest.mark.parametrize("family", MS.FAMILIES)
def test_hint_implies_may_pass_on_crafted_sets(lib, family):
    base = MS.generate(family, 200, f=525.0)
    tries = base + MS.variants(base)
    obj = np.stack([t.obj for t in tries])
    img = np.stack([t.img() for t in tries])
    for hint in HINTS:
        mp, hi, ac = _tries(lib, obj, img, 525.0, MS.PPX, MS.PPY, MS.TAU, hint)
        assert not (hi & ~mp).any(), (family, hint, [tries[i].params for i in np.flatnonzero(hi & ~mp)[:4]])
        assert not (ac & ~mp).any()
