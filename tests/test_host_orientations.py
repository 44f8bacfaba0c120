"""The device geometry at every camera orientation, not only within 30 degrees of the world axes (no GPU needed).

make_scene's own ground truths are rotations of at most 30 degrees; tests/orientations.py adds quarter turns, the approach
to a half turn, exact half turns (among them diag(1, -1, -1): y down, looking along world -z) and uniform draws.  These
tests run the host test hooks of libesac_b200.so -- the functions the kernels call -- at those orientations against cv2,
the 40-digit yardstick of tests/pose_loss_grid.py and the reference's own loss / dLoss, pinned in
tests/golden/pin/ref_pose_loss_edges.npz.
"""
import ast
import ctypes as C
from pathlib import Path

import cv2
import numpy as np
import pytest

import pose_loss_grid as G
from esac_b200.synth import make_scene, rodrigues
from oracle import esac_oracle as O
from oracle.build_ref import load_ref
from orientations import N_AXIS, NAMES, ORIENTATIONS, YZ_AXIS

GOLD = Path(__file__).resolve().parent / "golden"
PIN = GOLD / "pin" / "ref_pose_loss_edges.npz"
K = np.array([[525, 0, 320], [0, 525, 240], [0, 0, 1]], np.float64)


def _ptr(a):
    return a.ctypes.data


def _angle(Ra, Rb):
    """Angle between two rotations, atan2 form (exact near 0 and near pi)."""
    Rd = Ra @ Rb.T
    s = 0.5 * np.linalg.norm([Rd[2, 1] - Rd[1, 2], Rd[0, 2] - Rd[2, 0], Rd[1, 0] - Rd[0, 1]])
    return float(np.arctan2(s, (np.trace(Rd) - 1) / 2))


# ---- scenes --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", sorted(GOLD.glob("ref_*.npz")), ids=lambda p: p.stem)
def test_default_scenes_regenerate_every_fixture(path):
    """make_scene without `rotation` still draws every scene bit for bit as the fixtures were made."""
    z = np.load(path)
    kw = ast.literal_eval(str(z["scene_kw"]))
    sc = make_scene(**kw)
    assert np.array_equal(sc.assign, z["assign"])
    assert np.array_equal(sc.gt_pose, z["gt_pose"])
    if "coords" in z.files:
        assert np.array_equal(sc.coords, z["coords"])
    else:
        assert sc.coords.astype(np.float64).sum() == float(z["coords_sum"])


@pytest.mark.parametrize("name", ["pi_x", "pi_n", "uniform0"])
def test_rotation_argument_replaces_only_the_rotation(name):
    R = ORIENTATIONS[name]
    base = make_scene(E=2, H=12, W=16, M=8, seed=5)
    sc = make_scene(E=2, H=12, W=16, M=8, seed=5, rotation=R)
    assert np.array_equal(sc.assign, base.assign) and sc.gt_expert == base.gt_expert
    assert np.abs(sc.gt_pose[:3, :3].astype(np.float64) - R.T).max() < 1e-7
    assert np.array_equal(sc.gt_pose[:3, 3], base.gt_pose[:3, 3])   # the same camera centre
    r, _ = cv2.Rodrigues(R)
    by_rvec = make_scene(E=2, H=12, W=16, M=8, seed=5, rotation=r.ravel())
    assert np.abs(by_rvec.gt_pose - sc.gt_pose).max() < 1e-6
    # without noise and outliers the ground-truth expert's map is its camera's back-projection: every cell lies in front of
    # the rotated camera and reprojects onto its own pixel
    clean = make_scene(E=2, H=12, W=16, M=8, seed=5, rotation=R, noise=0.0, outlier_frac=0.0)
    X = clean.coords[clean.gt_expert].reshape(3, -1).T.astype(np.float64)
    Ti = np.linalg.inv(clean.gt_pose.astype(np.float64))
    xc = X @ Ti[:3, :3].T + Ti[:3, 3]
    assert (xc[:, 2] > 0.9).all()
    u = xc[:, 0] / xc[:, 2] * clean.f + clean.ppx
    v = xc[:, 1] / xc[:, 2] * clean.f + clean.ppy
    assert np.abs(u - np.tile(np.arange(16) * 8 + 4, 12)).max() < 1e-2
    assert np.abs(v - np.repeat(np.arange(12) * 8 + 4, 16)).max() < 1e-2


# ---- Rodrigues ---------------------------------------------------------------------------------------------------------
def _branch_edge_rotations():
    """Half-turn neighbours on both sides of rodrigues_m2v's s = 1e-5 branch (s = sin of the angle)."""
    out = {}
    for name, ax in (("n", N_AXIS), ("0,2,-3", YZ_AXIS), ("x", np.eye(3)[0])):
        for k, s in (("below", 0.99e-5), ("above", 1.01e-5)):
            out[f"edge_{k}_{name}"] = rodrigues(ax * (np.pi - np.arcsin(s)))
    return out


ROD_CASES = {**ORIENTATIONS, **_branch_edge_rotations()}


@pytest.mark.parametrize("name", list(ROD_CASES))
def test_rodrigues_both_ways_at_every_orientation(lib, name):
    R = ROD_CASES[name]
    rc, _ = cv2.Rodrigues(R)
    # vector -> matrix: bar 1e-12 against cv2 (and the jacobian)
    r = np.ascontiguousarray(rc.ravel())
    M = np.zeros(9); J = np.zeros(27)
    lib.esacb200_host_rodrigues(_ptr(r), _ptr(M), _ptr(J))
    Mc, Jc = cv2.Rodrigues(r.reshape(3, 1))
    assert np.abs(M.reshape(3, 3) - Mc).max() < 1e-12
    assert np.abs(J.reshape(3, 9) - Jc).max() < 1e-12 * max(1.0, np.abs(Jc).max())
    # matrix -> vector, compared as rotations (r and -r are the same rotation at pi): 1e-7 rad, the near-pi branch's precision
    back = np.zeros(3)
    lib.esacb200_host_rodrigues_inv(_ptr(np.ascontiguousarray(R.reshape(-1))), _ptr(back))
    Rb, _ = cv2.Rodrigues(back.reshape(3, 1))
    # the same rotation as cv2's vector, and no further from R than cv2's (within 2 sin(angle) of pi, OpenCV's branch takes
    # the axis from the diagonal alone and misses R by up to ~1e-5 rad: that is the reference's behaviour, kept)
    assert _angle(Rb, cv2.Rodrigues(rc)[0]) < 1e-7, (back, rc.ravel())
    assert _angle(Rb, R) <= _angle(cv2.Rodrigues(rc)[0], R) + 1e-7
    if not name.startswith("edge_below"):
        assert _angle(Rb, R) < 1e-7
    assert np.linalg.norm(back) <= np.pi + 1e-12


# ---- P3P ---------------------------------------------------------------------------------------------------------------
def _p3p_case(rng, R, noise):
    """4 scene points in front of a camera with world->camera rotation R, and their rounded pixels."""
    C0 = rng.uniform(-1, 1, 3)
    Xc = np.column_stack([rng.uniform(-1, 1, (4, 2)), rng.uniform(2, 4, 4)])
    X = ((Xc - 0) @ R + C0).astype(np.float32)                  # camera -> world: R^T xc + C
    t = -R @ C0
    xc = X.astype(np.float64) @ R.T + t
    uv = xc[:, :2] / xc[:, 2:] * 525 + np.array([320, 240])
    return np.ascontiguousarray(X), np.ascontiguousarray(np.round(uv + rng.normal(0, noise, uv.shape)).astype(np.float32))


def _fourth_point_error(X, uv, r, t):
    """Pixel distance of the 4th correspondence under pose (r, t): the criterion both P3P solvers pick their root by."""
    p, _ = cv2.projectPoints(X[3:4].astype(np.float64).reshape(1, 1, 3), np.reshape(r, (3, 1)), np.reshape(t, (3, 1)), K, None)
    return float(np.linalg.norm(p.ravel() - uv[3]))


@pytest.mark.parametrize("name", NAMES)
def test_p3p_matches_cv2_at_every_orientation(lib, name):
    """Same success and the same pose as solvePnP(P3P) on every try.  A different root is accepted only where it is a real
    tie: both roots bring the 4th point equally close (1e-6 px), so either is what the criterion picks."""
    rng = np.random.default_rng(NAMES.index(name) + 11)
    R = ORIENTATIONS[name]
    n_cmp = n_tie = 0
    for i in range(300):
        X, uv = _p3p_case(rng, R, (0.0, 1.0)[i % 2])
        ok, r1, t1 = cv2.solvePnP(X.reshape(-1, 1, 3), uv.reshape(-1, 1, 2), K, None, flags=cv2.SOLVEPNP_P3P)
        cv_ok = ok and not np.isnan(t1).any()
        pose = np.zeros(6); gate = C.c_int()
        mine = lib.esacb200_host_p3p_pose(_ptr(X), _ptr(uv), 525.0, 320.0, 240.0, 10.0, _ptr(pose), C.byref(gate))
        assert bool(mine) == bool(cv_ok)
        if not cv_ok:
            continue
        Rm, _ = cv2.Rodrigues(pose[:3].reshape(3, 1))
        Rc, _ = cv2.Rodrigues(r1)
        assert abs(np.linalg.det(Rm) - 1) < 1e-9   # a proper rotation, never a reflection
        d = _angle(Rm, Rc) + np.abs(pose[3:] - t1.ravel()).max()
        if d < 1e-8:
            n_cmp += 1
            continue
        e_mine, e_cv = _fourth_point_error(X, uv, pose[:3], pose[3:]), _fourth_point_error(X, uv, r1, t1)
        assert abs(e_mine - e_cv) < 1e-6, (i, d, e_mine, e_cv)
        n_tie += 1
    assert n_cmp > 250 and n_tie <= 3, (n_cmp, n_tie)


# ---- the float prefilter ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pi_x", "pi_0,2,-3", "179.99_n", "uniform1"])
def test_float_prefilter_never_rejects_an_accepted_try_at_any_orientation(lib, name):
    """p3p_may_pass uses distances and bearings only, so its guarantee cannot depend on the camera's orientation."""
    sc = make_scene(E=2, H=60, W=80, M=8, sub=8, seed=1, rotation=ORIENTATIONS[name])
    pl = sc.coords[sc.gt_expert]
    rng = np.random.default_rng(5)
    mp_, ac, ev = C.c_int(), C.c_int(), C.c_int()
    n_acc = 0
    for _ in range(20000):
        while True:
            xs = rng.integers(0, 79, 4); ys = rng.integers(0, 59, 4)
            if len({(a, b) for a, b in zip(xs, ys)}) == 4:
                break
        obj = np.ascontiguousarray(pl[:, ys, xs].T.astype(np.float32))
        img = np.ascontiguousarray(np.stack([xs * 8 + 4, ys * 8 + 4], 1).astype(np.float32))
        lib.esacb200_host_try(_ptr(obj), _ptr(img), sc.f, sc.ppx, sc.ppy, sc.tau, 2.0, C.byref(mp_), C.byref(ac))
        assert not (ac.value and not mp_.value)
        pv = np.zeros(6)
        lib.esacb200_host_try_verdict(_ptr(obj), _ptr(img), sc.f, sc.ppx, sc.ppy, sc.tau, C.byref(ev), _ptr(pv))
        assert ev.value == ac.value
        if ac.value:
            pf = np.zeros(6); gate = C.c_int()
            lib.esacb200_host_p3p_pose(_ptr(obj), _ptr(img), sc.f, sc.ppx, sc.ppy, sc.tau, _ptr(pf), C.byref(gate))
            assert np.array_equal(pv, pf)
            Rp, _ = cv2.Rodrigues(pf[:3].reshape(3, 1))
            n_acc += _angle(Rp, ORIENTATIONS[name]) < np.radians(5)
    assert n_acc > 500   # exercised on accepted tries, whose poses are the rotated camera's


# ---- loss / dLoss --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pin():
    return np.load(PIN)


@pytest.mark.parametrize("name", NAMES)
def test_host_loss_and_dloss_at_every_orientation(lib, pin, name):
    gt = G.ground_truth(name)
    gt64 = np.ascontiguousarray(gt.astype(np.float64).ravel())
    r2, t2 = O.trans2pose(gt.astype(np.float64))
    gt6 = np.ascontiguousarray(np.concatenate([r2.ravel(), t2.ravel()]))
    poses, _ = G.estimates(gt)
    cuts = pin[f"{name}_cuts"]
    losses, dloss = np.zeros(len(poses)), np.zeros((len(poses), 6))
    for i, est in enumerate(poses):
        est = np.ascontiguousarray(est)
        T1 = np.zeros(16)
        lib.esacb200_host_pose2trans(_ptr(est), _ptr(T1))
        losses[i] = lib.esacb200_host_loss(_ptr(T1), _ptr(gt64), G.W_ROT, G.W_TRANS, cuts[i])
        d = np.zeros(6)
        lib.esacb200_host_dloss(_ptr(est), _ptr(gt6), G.W_ROT, G.W_TRANS, cuts[i], _ptr(d))
        dloss[i] = d
    G.check_pose_loss(name, losses, dloss, pin)


def test_oracle_dloss_returns_what_the_reference_returns_at_a_clamped_trace(pin):
    """Where the trace clamps to 3 or -1, dLoss's -1/sqrt(0) = -inf meets the zeros of dTrace first, so the reference's NaN
    check returns zeros, never +-inf.  Every component of the oracle's dLoss must fall in a class the pinned reference
    returns at that entry, and at entries the reference answers with a single class, in that class."""
    n_zero = 0
    for name in NAMES:
        gt64 = G.ground_truth(name).astype(np.float64)
        r2, t2 = O.trans2pose(gt64)
        for est, cut, ref, allowed in zip(pin[f"{name}_poses"], pin[f"{name}_cuts"], pin[f"{name}_dloss"], pin[f"{name}_class"]):
            d = O.d_loss(est[:3], est[3:], r2, t2, G.W_ROT, G.W_TRANS, cut).ravel()
            assert np.all(G.classes(d) & allowed), (name, est, d, ref, allowed)
            assert not np.any(allowed & G.CLASS_NONFINITE)
            n_zero += bool(np.all(d == 0) and np.all(ref == 0))
    assert n_zero > 100


def test_reference_binding_reproduces_the_pose_loss_pin(pin):
    R = load_ref()
    if R is None:
        pytest.skip("oracle/_ref is not built and no readable reference checkout was found (oracle/build_ref.py)")
    import sys
    sys.path.insert(0, str(GOLD))
    from make_ref_pose_loss_pin import pin_orientation
    for name in NAMES:
        got = pin_orientation(R, name)
        for k, v in got.items():
            assert np.array_equal(v, pin[k], equal_nan=True), k
