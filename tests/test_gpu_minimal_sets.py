"""The sampling stage's device verdicts on crafted minimal sets (tests/minimal_sets.py), run with `-m gpu` on an H100.

Every crafted try is injected as try 0 of its own hypothesis, with its plane's anchor set as try 1, into one forward of
~75k hypotheses on 64 planes of 60 x 80 cells (sub = 8), so each call judges every crafted try once on the device compile
of the prefilter (sqrt.approx, __fdividef, MUFU rsqrt, contracted FMAs) and of the exact path.  Under the default
schedule (waves: prefilter_kernel + exact_kernel), sample_prefilter = 0, sample_waves = 0 (every try in tail_kernel, the
other compile of the prefilter) and sample_groups 1 and 4, tries, cells and poses must be bitwise equal; every crafted
verdict (tries == 1) must equal the cv2 oracle's, except rounding ties shown at 40 digits (minimal_sets.rounding_tie);
every anchor must pass; and accepted tries must reproject their 4 points like the oracle's pose does."""
import cv2
import numpy as np
import pytest

import minimal_sets as MS
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

E_PLANES = 64
N_BASE = 1100      # per family at f = 525: x 11 variants x 6 families ~ 73k hypotheses per call
POSE_TOL = 1e-8    # test_gpu_sample_schedules.py, on the well-conditioned family
ALPHA, BETA, MAX_REPROJ = 100.0, 0.5, 100.0
SCHEDULES = {"default": {}, "no_prefilter": {"sample_prefilter": 0}, "tail_only": {"sample_waves": 0},
             "groups1": {"sample_groups": 1}, "groups4": {"sample_groups": 4}}
DEFAULTS = {"sample_prefilter": 1, "sample_waves": 6, "sample_groups": 2, "fixed_seed": 0}


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    return api


def _tagged(family, n, f):
    """Base tries and their variants, each tagged with the index of its base try."""
    out = []
    for i, t in enumerate(MS.generate(family, n, seed=11, f=f)):
        for v in [t] + MS.variants([t]):
            v.params = dict(v.params, base=(family, i))
            out.append(v)
    return out


def _run(api, pk, f, opts):
    ctx = api.context()
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        api.set_seed(5)
        api.inject_cells(pk.cells)
        out = np.zeros((4, 4), np.float32)
        api.forward(pk.coords, pk.assign, out, 0, 0, f, MS.PPX, MS.PPY, MS.TAU, ALPHA, BETA, MAX_REPROJ, MS.SUB)
        return api.last_hypotheses(), ctx.sample_profile()
    finally:
        ctx.inject_cells(None)
        for k, v in DEFAULTS.items():
            ctx.set_option(k, v)


def _reproj(pose, obj, img, K):
    proj, _ = cv2.projectPoints(obj.reshape(-1, 1, 3), pose[:3].reshape(3, 1), pose[3:].reshape(3, 1), K, None)
    return np.linalg.norm(img.astype(np.float64) - proj.reshape(-1, 2), axis=1)


@pytest.fixture(scope="module", params=[525.0, 3000.0], ids=["f525", "f3000"])
def crafted(request, api):
    f = request.param
    fams = MS.FAMILIES if f == 525.0 else ("parallel",)
    tries = [t for fam in fams for t in _tagged(fam, N_BASE if f == 525.0 else 2000, f)]
    pk = MS.pack(tries, E_PLANES, f)
    runs = {name: _run(api, pk, f, opts) for name, opts in SCHEDULES.items()}
    K = O.cam_mat(f, MS.PPX, MS.PPY)
    ref = O.sample_hypotheses(pk.coords, pk.assign, O.create_sampling(MS.W, MS.H, MS.SUB, 0, 0), K, 10 ** 6, MS.TAU,
                              injected_cells=pk.cells)
    return f, pk, runs, ref, K


def test_schedules_agree_bitwise(crafted):
    _, pk, runs, _, _ = crafted
    base = runs["default"][0]
    for name, (hy, prof) in runs.items():
        print(name, prof)
        for key in ("tries", "cells", "poses"):
            bad = np.flatnonzero((hy[key] != base[key]).reshape(len(pk.tries), -1).any(axis=1))
            assert bad.size == 0, (name, key, bad[:8])


def test_crafted_verdicts_match_the_oracle(api, crafted):
    f, pk, runs, ref, K = crafted
    hy = runs["default"][0]
    dev_acc = hy["tries"] == 1
    ref_acc = np.array([h.tries == 1 for h in ref])
    lib = api.load_library()
    stats = {}
    bad = []
    for h in range(len(pk.tries)):
        t = pk.tries[h]
        s = stats.setdefault(t.family, [0, 0, 0])
        s[0] += 1
        s[1] += bool(dev_acc[h])
        if dev_acc[h] != ref_acc[h]:
            if MS.rounding_tie(MS.root_errors(lib, t.obj, t.img(), f)):
                s[2] += 1
            else:
                bad.append(h)
    for fam, (n, acc, tie) in stats.items():
        print(f"f={f:g} {fam}: {n} crafted tries, {acc} accepted, {tie} rounding ties excused")
    assert not bad, [(pk.tries[h].params, bool(dev_acc[h])) for h in bad[:5]]
    assert 0 < dev_acc.sum() < len(dev_acc)


def test_anchors_pass_and_accepted_poses_reproject_like_the_oracle(api, crafted):
    f, pk, runs, ref, K = crafted
    hy = runs["default"][0]
    anc = MS.anchor_obj(f)
    anc_img = (np.array(MS.ANCHOR_CELLS) * MS.SUB + MS.SUB // 2).astype(np.float32)
    assert np.all(hy["tries"] <= 2)
    for h in np.flatnonzero(hy["tries"] == 2):   # the crafted try failed: the anchor must have passed
        assert _reproj(hy["poses"][h], anc, anc_img, K).max() < MS.TAU, h
    n_pose = 0
    for h in np.flatnonzero((hy["tries"] == 1) & np.array([r.tries == 1 for r in ref])):
        t, r = pk.tries[h], ref[h]
        ref_pose = np.concatenate([r.rvec.ravel(), r.tvec.ravel()])
        e_dev, e_ref = _reproj(hy["poses"][h], t.obj, t.img(), K), _reproj(ref_pose, t.obj, t.img(), K)
        # P3P fits its three points exactly: the device pose puts them on their pixels to the float32 rounding.  cv2's
        # fp64 pose is not always as accurate (up to ~0.1 px off them near the danger cylinder at the 1e5 m offset, where
        # its solver works on uncentred coordinates), so the 4th point is held to 1e-4 px plus twice the misfit cv2's
        # pose shows on the three points it solved.
        assert e_dev[:3].max() < 1e-4, (t.params, e_dev)
        agree = np.abs(e_dev - e_ref).max() < 1e-4 + 2 * e_ref[:3].max()
        if not agree and MS.rounding_tie(MS.root_errors(api.load_library(), t.obj, t.img(), f)):
            continue   # two roots tie on the 4th point: either pose is the reference's
        assert agree, (t.params, e_dev, e_ref)
        if t.family == "noise" and "scale" not in t.params and "offset" not in t.params:
            assert np.abs(hy["poses"][h] - ref_pose).max() < POSE_TOL, t.params
            n_pose += 1
    assert n_pose > 100 or "noise" not in {t.family for t in pk.tries}


def test_prefilter_rejected_some_of_the_crafted_tries(crafted):
    """Both sides of the prefilter ran on crafted tries: without it every try is judged exactly (2 per hypothesis: the
    crafted set and, where it fails, the anchor), with it fewer.  The crafted 4th points all lie within 1.2 tau of the true
    pose, inside the 2 tau band, so the prefilter may pass most of them; what it rejects are sets whose other roots miss."""
    _, pk, runs, _, _ = crafted
    judged = runs["default"][1]["survivors_judged"]
    judged_all = runs["no_prefilter"][1]["survivors_judged"]
    print("tries judged exactly:", judged, "of", judged_all)
    assert judged_all >= len(pk.tries)
    assert 0 < judged < judged_all


def test_power_of_two_scales_are_exact(crafted):
    """The fp64 path is equivariant under 2^k scales (tests/test_host_minimal_sets.py): the same verdict and rvec, the
    tvec scaled by exactly 2^k."""
    _, pk, runs, _, _ = crafted
    hy = runs["default"][0]
    where = {(t.params["base"], t.params.get("scale"), t.params.get("offset")): h for h, t in enumerate(pk.tries)}
    n = 0
    for (base, s, off), h in where.items():
        if s is None or off is not None or np.log2(s) != np.round(np.log2(s)) or (base, None, None) not in where:
            continue
        b = where[(base, None, None)]
        assert hy["tries"][h] == hy["tries"][b], (base, s)
        if hy["tries"][h] == 1:
            assert np.array_equal(hy["poses"][h][:3], hy["poses"][b][:3]) and \
                np.array_equal(hy["poses"][h][3:], hy["poses"][b][3:] * s), (base, s)
            n += 1
    assert n > 100
