"""The sampling stage's verdicts on crafted minimal sets (tests/minimal_sets.py), on the host compile of its code.  No GPU.

For every try: the float prefilter (p3p_may_pass_fast) never rejects a try the exact fp64 path accepts, the verdict path
(early exit at 1.25 tau + 1 px) gives the full path's verdict, and the exact verdict equals the cv2 oracle's gate
(safe_solve_pnp + projectPoints, as oracle.esac_oracle.sample_hypotheses runs it).  A verdict that differs from cv2's is
excused only where a 40-digit solve shows a rounding tie (minimal_sets.rounding_tie)."""
import ctypes as C

import cv2
import numpy as np
import pytest

import minimal_sets as MS
from oracle import esac_oracle as O

MARGIN = 2.0   # kPrefilterMargin, the shipping band
# base tries per family (each also scaled and offset: x11); the danger cylinder fails rarely, so it gets the most
N_BASE = {"cylinder": 1000, "needle": 200, "parallel": 200, "flat": 200, "spread": 200, "noise": 200}
CASES = [(fam, 525.0) for fam in MS.FAMILIES] + [("parallel", 3000.0)]


def cv2_verdict(obj, img, f):
    K = O.cam_mat(f, MS.PPX, MS.PPY)
    ok, r, t = O.safe_solve_pnp(obj, img, K, None, None, False, cv2.SOLVEPNP_P3P)
    if not ok:
        return False
    proj, _ = cv2.projectPoints(obj.reshape(-1, 1, 3), r, t, K, None)
    d = img - proj.reshape(-1, 2).astype(np.float32)
    return bool(np.all(np.sqrt(d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2) < MS.TAU))


def host_verdicts(lib, t):
    """(may_pass, exact accept, verdict-path accept, pose of the verdict path) of one try on the host compile."""
    obj, img = np.ascontiguousarray(t.obj), np.ascontiguousarray(t.img())
    mp, ac, ev = C.c_int(), C.c_int(), C.c_int()
    lib.esacb200_host_try(obj.ctypes.data, img.ctypes.data, t.f, MS.PPX, MS.PPY, MS.TAU, MARGIN, C.byref(mp), C.byref(ac))
    pv = np.zeros(6)
    lib.esacb200_host_try_verdict(obj.ctypes.data, img.ctypes.data, t.f, MS.PPX, MS.PPY, MS.TAU, C.byref(ev), pv.ctypes.data)
    return bool(mp.value), bool(ac.value), bool(ev.value), pv


@pytest.mark.parametrize("family,f", CASES)
def test_crafted_sets_prefilter_and_verdicts(lib, family, f):
    base = MS.generate(family, N_BASE[family], f=f)
    tries = base + MS.variants(base)
    false_rejects, verdict_diffs, cv2_diffs = [], [], []
    n_acc = n_may = n_excused = 0
    for t in tries:
        may, acc, ver, _ = host_verdicts(lib, t)
        n_acc += acc
        n_may += may
        if acc and not may:
            false_rejects.append(t)
        if ver != acc:
            verdict_diffs.append(t)
        if cv2_verdict(t.obj, t.img(), f) != acc:
            if MS.rounding_tie(MS.root_errors(lib, t.obj, t.img(), f)):
                n_excused += 1
            else:
                cv2_diffs.append(t)
    print(f"{family} f={f:g}: {len(tries)} tries, {n_acc} accepted, {n_may} sent to the exact path, "
          f"{n_excused} rounding ties excused")
    assert not false_rejects, f"{len(false_rejects)} accepted tries rejected by the prefilter, e.g. " \
                              f"{false_rejects[0].params} obj={false_rejects[0].obj.tolist()} cells={false_rejects[0].cells.tolist()}"
    assert not verdict_diffs, f"{len(verdict_diffs)} verdict-path decisions differ, e.g. {verdict_diffs[0].params}"
    assert not cv2_diffs, f"{len(cv2_diffs)} exact verdicts differ from cv2's, e.g. {cv2_diffs[0].params}"
    assert 0 < n_acc < len(tries)   # both verdicts were exercised


def test_issue_reproducer_is_not_rejected(lib):
    """A near-cylinder set whose first three points are noise-free: the exact path and cv2 accept it (4th point 2.08 px
    off), the float prefilter used to reject it at any margin below 1000 tau."""
    obj = np.array([[1.9387993812561035, -1.769748330116272, 4.7974138259887695],
                    [0.7416813969612122, -0.4984383285045624, 1.2304093837738037],
                    [-3.8788952827453613, 6.716091632843018, 27.886783599853516],
                    [-0.6180092692375183, 0.25266051292419434, 1.3614336252212524]], np.float32)
    img = np.array([[532.1704711914062, 46.329437255859375], [636.4660034179688, 27.32271385192871],
                    [246.97544860839844, 366.4379577636719], [80.58016204833984, 338.1081848144531]], np.float32)
    mp, ac = C.c_int(), C.c_int()
    lib.esacb200_host_try(obj.ctypes.data, img.ctypes.data, 525.0, 320.0, 240.0, 10.0, MARGIN, C.byref(mp), C.byref(ac))
    assert ac.value and cv2_verdict(obj, img, 525.0)
    assert mp.value


def test_exact_path_is_equivariant_under_power_of_two_scales(lib):
    """Scaling the scene by 2^k is exact in float32; the fp64 path must give the same verdict, the same rvec and a tvec
    scaled by exactly 2^k (tests/test_gpu_minimal_sets.py relies on it)."""
    n = 0
    for fam in MS.FAMILIES:
        for t in MS.generate(fam, 60, seed=7):
            _, acc, _, pose = host_verdicts(lib, t)
            for k in (-40, -20, -10, 10, 20, 40):
                s = 2.0 ** k
                o = (t.obj.astype(np.float64) * s).astype(np.float32)
                if not MS._normal(o):
                    continue
                _, acc_s, _, pose_s = host_verdicts(lib, MS.Try(t.family, t.f, t.cells, o))
                assert acc_s == acc
                if acc:
                    assert np.array_equal(pose_s[:3], pose[:3]) and np.array_equal(pose_s[3:], pose[3:] * s), (fam, k)
                    n += 1
    assert n > 500
