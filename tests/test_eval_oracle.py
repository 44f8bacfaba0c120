"""The evaluation oracle (oracle/eval_oracle.py) against the reference's own route on the same float32 inputs
(test_esac.py:209-247: a float32 numpy product, cv2.Rodrigues, a float32 torch.norm, torch's inverse), and its table
against hand-worked cases.  No GPU.

Tolerances come from float32 rounding on the reference's side.  The entries of its float32 product P_R G_R^T carry errors of
a few 1e-8 each, so the cosine c that Rodrigues takes the angle from is off by at most dc = 1e-6 (generous); the angle is
then off by at most dc / sin(theta), and never more than sqrt(2 dc) where acos is ill-conditioned (near 0 and near 180
degrees).  The translation error is a float32 norm of a float32 difference: 1e-6 relative.  The inverse's translation is
float32 too: 1e-6 of (1 + |t|) in each component."""
import math

import cv2
import numpy as np
import pytest
import torch

from oracle import eval_oracle as O
from orientations import cam_to_world, rotate, uniform_rotations

DC = 1e-6


def reference_route(out_pose: np.ndarray, gt_pose: np.ndarray):
    """test_esac.py:209-247 verbatim in its types: (rot_deg, trans_cm, rvec is zero, q [4], t [3])."""
    out_t, gt_t = torch.from_numpy(out_pose), torch.from_numpy(gt_pose)
    t_err = float(torch.norm(gt_t[0:3, 3] - out_t[0:3, 3]))
    r_err = np.matmul(out_pose[0:3, 0:3], np.transpose(gt_pose[0:3, 0:3]))
    r_err = cv2.Rodrigues(r_err)[0]
    zero = not np.any(r_err)
    r_err = np.linalg.norm(r_err) * 180 / math.pi
    inv = out_t.inverse()
    t = inv[0:3, 3]
    rot, _ = cv2.Rodrigues(inv[0:3, 0:3].numpy())
    angle = np.linalg.norm(rot)
    with np.errstate(invalid="ignore", divide="ignore"):
        axis = rot / angle
    q = np.concatenate([[math.cos(angle * 0.5)], (math.sin(angle * 0.5) * axis).reshape(3)])
    return r_err, t_err * 100, zero, q, t.numpy().astype(np.float64)


def _pose(R, centre=(0.3, -0.2, 1.5)):
    return cam_to_world(np.asarray(R, np.float64), centre)


def _pairs():
    rng = np.random.default_rng(7)
    rots = uniform_rotations(80, seed=31)
    pairs = [("uniform", _pose(rots[i]), _pose(rots[i + 1], rng.uniform(-3, 3, 3))) for i in range(0, 80, 2)]
    for k, R in enumerate(uniform_rotations(12, seed=5)):
        axis = rng.normal(size=3)
        for ang in (0.8e-5, 1.2e-5):
            pairs.append((f"straddle {ang}", _pose(rotate(R, axis, ang)), _pose(R)))
        pairs.append(("identity", _pose(R), _pose(R)))
        for deg in (179.0, 179.5, 179.9, 180.0):
            pairs.append((f"half turn {deg}", _pose(rotate(R, axis, math.radians(deg))), _pose(R)))
        far = rng.uniform(-1, 1, 3)
        far *= 1000.0 / np.linalg.norm(far)
        pairs.append(("1 km", _pose(rots[k], far), _pose(rots[k + 1], far + rng.uniform(-2, 2, 3))))
        skew = _pose(rots[k])
        skew[:3, :3] += rng.uniform(-3e-4, 3e-4, (3, 3)).astype(np.float32)   # slightly non-orthonormal
        pairs.append(("non-orthonormal", skew, _pose(rots[k + 2])))
    return pairs


PAIRS = _pairs()


@pytest.mark.parametrize("kind", sorted({k for k, _, _ in PAIRS}))
def test_oracle_matches_reference_route(kind):
    for _, P, G in (p for p in PAIRS if p[0] == kind):
        rec = O.evaluate(P, G, expert=2, scene=2)
        r_ref, t_ref, zero_ref, q_ref, tvec_ref = reference_route(P, G)
        theta = math.radians(rec[0])
        tol = min(DC / max(math.sin(theta), 1e-300), math.sqrt(2 * DC)) + 1e-7
        assert abs(math.radians(r_ref) - theta) <= tol, (kind, r_ref, rec[0])
        # the exact-zero branch agrees wherever s is not within 1e-6 of the threshold
        X = O.polar_newton((P[:3, :3].astype(np.float64) @ G[:3, :3].astype(np.float64).T).reshape(9))
        _, s, c = O.rodrigues_sin_cos(X)
        if abs(s - 1e-5) > 1e-6 and c > 0:
            assert (rec[0] == 0.0) == zero_ref, (kind, s, rec[0], r_ref)
        assert abs(t_ref - rec[1]) <= 1e-6 * max(rec[1], 1e-3), (kind, t_ref, rec[1])
        assert np.abs(tvec_ref - rec[11:14]).max() <= 1e-6 * (1 + np.linalg.norm(rec[11:14])), (kind, tvec_ref, rec[11:14])
        if np.isnan(q_ref[1:]).any():
            assert np.isnan(rec[8:11]).all() and q_ref[0] == rec[7] == 1.0
        else:  # q and -q are one rotation: at 180 degrees the axis' sign is a rounding decision
            dq = min(np.abs(q_ref - rec[7:11]).max(), np.abs(q_ref + rec[7:11]).max())
            assert dq <= 2e-3 if kind.startswith("half turn") else dq <= 1e-5, (kind, q_ref, rec[7:11])


def test_straddling_angles_fall_on_both_sides_of_the_zero_branch():
    R = uniform_rotations(1, seed=3)[0]
    small = O.evaluate(_pose(rotate(R, (0, 0, 1), 0.8e-5)), _pose(R), 0, 0)
    large = O.evaluate(_pose(rotate(R, (0, 0, 1), 1.2e-5)), _pose(R), 0, 0)
    assert small[0] == 0.0 and large[0] > 0.0


def test_pose_file_quaternion_is_nan_at_angle_zero():
    P = np.eye(4, dtype=np.float32)
    P[:3, 3] = (1.0, 2.0, 3.0)
    rec = O.evaluate(P, P, 0, 0)
    assert rec[7] == 1.0 and np.isnan(rec[8:11]).all()
    assert np.array_equal(rec[11:14], [-1.0, -2.0, -3.0])
    assert O.pose_line("seq-01/frame-000000", rec) == "seq-01/frame-000000 1.000000 nan nan nan -1.000000 -2.000000 -3.000000"
    _, _, _, q_ref, _ = reference_route(P, P)
    assert np.isnan(q_ref[1:]).all()


def _rec(rot, trans, scene, expert, status=0, active=1.0):
    r = np.zeros(14)
    r[:7] = (rot, trans, float(scene == expert), scene, expert, status, active)
    return r


def test_table_upper_median_empty_scene_and_average():
    recs = [_rec(1.0, 2.0, 0, 0), _rec(4.0, 8.0, 0, 0), _rec(3.0, 6.0, 0, 1), _rec(2.0, 4.0, 0, 0),   # scene 0: 4 images
            _rec(7.0, 1.0, 2, 2, active=3.0)]                                                          # scene 2: 1; scene 1: none
    t = O.table(recs, 3)
    # scene 0: rot sorted 1 2 3 4 -> [2] = 3; trans 2 4 6 8 -> 6; class 3/4; pose (t < 5 and r < 5): 2/4
    assert t["console"][2] == "%7d %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (0, 75.0, 50.0, 3.0, 6.0)
    assert t["console"][3] == "%7d %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (1, 0.0, 0.0, 0, 0)
    assert t["console"][4] == "%7d %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (2, 100.0, 0.0, 7.0, 1.0)
    assert t["results"] == ["0.750000 0.500000 3.000000 6.000000", "0.000000 0.000000 0.000000 0.000000",
                            "1.000000 0.000000 7.000000 1.000000"]
    # the Average row divides by the 3 scenes, the empty one included
    assert t["console"][-1] == "Average %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (175 / 3, 50 / 3, 10 / 3, 7 / 3)
    assert t["experts"] == ["Avg. experts active: 1.4", "Max. experts active: 3.0"]
    assert t["excluded"] == 0
    assert O.table(recs, 3, average=False)["console"][-1] == t["console"][4]


def test_table_thresholds_are_strict():
    recs = [_rec(5.0, 1.0, 0, 0), _rec(1.0, 5.0, 0, 0), _rec(4.999999, 4.999999, 0, 0)]
    t = O.table(recs, 1)
    assert t["results"][0].split()[1] == "%f" % (1 / 3)
    t = O.table(recs, 1, rot_threshold=5.0000001, trans_threshold=5.0000001)
    assert t["results"][0].split()[1] == "%f" % 1.0


def test_table_leaves_out_failed_forwards_and_foreign_scenes():
    recs = [_rec(1.0, 1.0, 0, 0), _rec(np.nan, np.nan, 0, -1, status=1, active=4.0), _rec(1.0, 1.0, 5, 5),
            _rec(1.0, 1.0, -1, 0), _rec(3.0, 3.0, 0, 0)]
    t = O.table(recs, 2)
    assert t["excluded"] == 3
    assert t["results"][0] == "1.000000 1.000000 3.000000 3.000000"
    assert t["experts"] == ["Avg. experts active: 1.0", "Max. experts active: 1.0"]


def test_product_table_equals_oracle_table():
    """esac_b200.evaluate's table (the one PoseEvaluator.table formats) against the oracle's on random records."""
    from esac_b200.evaluate import _table
    rng = np.random.default_rng(3)
    recs = np.stack([_rec(rng.uniform(0, 10), rng.uniform(0, 10), int(rng.integers(-1, 6)), int(rng.integers(0, 5)),
                          status=int(rng.random() < 0.1), active=float(rng.integers(1, 5))) for _ in range(301)])
    for avg in (True, False):
        a, b = _table(recs, 5, 5, 5, avg), O.table(recs, 5, average=avg)
        assert (a["console"], a["results"], a["experts"], a["excluded"]) == (b["console"], b["results"], b["experts"],
                                                                             b["excluded"])
