"""The pose-loss edge grid of the orientation tests, and its 40-digit yardstick.

For every ground-truth orientation of tests/orientations.py, estimates sit at rotation distances from exactly 0 to exactly
pi and translation distances from 0 to 1e7, under three cuts: off, on, and equal to the loss.  `yardstick` evaluates the
reference's loss() and dLoss() (esac_loss.h, quirks included: PI = 3.1415926 in loss(), CV_PI in dLoss(), dLoss's cut
branch scaled by 0.5 / sqrt(loss)) in mpmath on the float64 inputs, with the ground truth's rotation taken as the exact
polar factor of the float32 matrix (what cv::Rodrigues makes of it).

Where float64 cannot resolve what the formulas do, there is no value to compare: the clamped trace (rotation distance
within about 1e-7 of 0 or pi, where dLoss divides by sqrt(0)), tErr = 0 (0 / 0), the MAXLOSS exit.  `degenerate` flags
those entries; there the tests compare the outcome class (zero, finite, non-finite) with what the compiled reference
returns (tests/golden/pin/ref_pose_loss_edges.npz).

Elsewhere a value must lie within 4x the float64 oracle's distance from the yardstick plus 1e-12 relative plus a floor of
what float64 cannot know (`yardstick`).  The widest part of that floor is the ground truth's rotation: float64 recovers it
from the float32 matrix only to Truth.delta = 64 u / sin(angle), with sin clamped at 1e-5, and the translation error's
direction amplifies that by |invT2| / tErr (about 1.5e6 at tErr = 1e-6).  So at the half-turn ground truths with the
1e-6 translation each dLoss component is held only to about 2e-3 of its size; at 179.99 degrees about 1e-4; at tErr = 1
or at orientations away from a half turn below 1e-7.  Those entries check the branch taken and the formula, not the last
digits.
"""
import cv2
import mpmath as mp
import numpy as np

from oracle import esac_oracle as O
from orientations import ORIENTATIONS, cam_to_world, half_turn, rotate

ROT_DIST = {"0": 0.0, "1e-9": 1e-9, "1e-6": 1e-6, "1e-3": 1e-3, "1deg": np.radians(1.0), "30deg": np.radians(30.0),
            "90deg": np.radians(90.0), "170deg": np.radians(170.0), "179.9deg": np.radians(179.9), "pi-1e-6": np.pi - 1e-6,
            "pi": np.pi}
TRANS_DIST = (0.0, 1e-6, 1.0, 1e7)
CUTS = ("off", "on", "equal")
W_ROT, W_TRANS = 1.0, 100.0
CUT_OFF, CUT_ON = 1e30, 1.0
TURN_AXIS = np.array([-2.0, 1.0, 0.5]) / np.sqrt(5.25)   # the axis the estimates turn about, away from the ground truth
SHIFT_DIR = np.array([2.0, -1.0, 2.0]) / 3.0             # the direction their camera centres move in
MAXLOSS = 10000000.0
EPS = 0.00000001
PI_LOSS = mp.mpf(3.1415926)
CLASS_ZERO, CLASS_FINITE, CLASS_NONFINITE = 1, 2, 4


def polar(M):
    U, _, Vt = np.linalg.svd(np.asarray(M, np.float64))
    return U @ Vt


def ground_truth(name):
    """float32 camera->world ground truth of orientation `name`."""
    return cam_to_world(ORIENTATIONS[name])


def estimates(gt):
    """The grid around one ground truth: poses float64 [N, 6] (rvec, tvec: scene poses, what esac's hypotheses are),
    and per entry its (rotation distance name, translation distance, cut name)."""
    R0 = polar(gt[:3, :3].astype(np.float64)).T   # world->camera
    C0 = gt[:3, 3].astype(np.float64)
    poses, keys = [], []
    for dname, d in ROT_DIST.items():
        R = half_turn(TURN_AXIS) @ R0 if dname == "pi" else rotate(R0, TURN_AXIS, d)
        r, _ = cv2.Rodrigues(R)
        for dt in TRANS_DIST:
            C = C0 + dt * SHIFT_DIR
            for cut in CUTS:
                poses.append(np.concatenate([r.ravel(), -R @ C]))
                keys.append((dname, dt, cut))
    return np.array(poses), keys


# ---------------------------------------------------------------------------------------------------------------------
# 40-digit restatement
# ---------------------------------------------------------------------------------------------------------------------
def _rod(r):
    th = mp.sqrt(r[0] ** 2 + r[1] ** 2 + r[2] ** 2)
    if th == 0:
        return mp.eye(3)
    k = [x / th for x in r]
    K = mp.matrix([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return mp.eye(3) + mp.sin(th) * K + (1 - mp.cos(th)) * (K * K)


def _drod(r):
    """d vec(R) / d r, 3 x 9 (cv::Rodrigues' jacobian layout), by central differences at 40 digits (error ~1e-25)."""
    h = mp.mpf("1e-15")
    out = mp.matrix(3, 9)
    for i in range(3):
        rp = list(r); rm = list(r)
        rp[i] += h; rm[i] -= h
        D = (_rod(rp) - _rod(rm)) / (2 * h)
        for k in range(9):
            out[i, k] = D[k // 3, k % 3]
    return out


def _polar_mp(M):
    X = M.copy()
    for _ in range(12):
        X = (X + mp.inverse(X).T) / 2
    return X


class Truth:
    """The ground truth `gt` (float32 4x4 camera->world) in 40 digits: raw transform, and the scene pose dLoss sees."""

    def __init__(self, gt):
        with mp.workdps(40):
            self.T = mp.matrix([[mp.mpf(float(v)) for v in row] for row in gt.astype(np.float64)])
            Rc = self.T[:3, :3]
            Ri = mp.inverse(Rc)                        # rotation block of trans.inv()
            self.R2 = _polar_mp(Ri)                    # what cv::Rodrigues makes of it
            tt = mp.matrix([self.T[0, 3], self.T[1, 3], self.T[2, 3]])
            self.t2 = -(Ri * tt)
            # float64 knows the ground truth's rotation (cv::Rodrigues' vector of it) only to about u / sin(angle): near a
            # half turn the vector comes from a small antisymmetric part, or from the diagonal alone
            R2 = self.R2
            sin = mp.sqrt((R2[2, 1] - R2[1, 2]) ** 2 + (R2[0, 2] - R2[2, 0]) ** 2 + (R2[1, 0] - R2[0, 1]) ** 2) / 2
            self.delta = 64 * mp.mpf(2) ** -52 / max(sin, mp.mpf("1e-5"))


TRACE_SLACK = 16 * 2.0 ** -52 * 4   # 16 units in the last place of a trace near 3: how far float64 sums may move it


def _rot_err(tr, pi):
    tr = min(mp.mpf(3), max(mp.mpf(-1), tr))
    return 180 * mp.acos((tr - 1) / 2) / pi


def _coef(tr):
    tr = min(mp.mpf(3), max(mp.mpf(-1), tr))
    den = 3 - tr * tr + 2 * tr
    return (180 / mp.pi) * -1 / mp.sqrt(den) if den > 0 else None


def yardstick(est, truth: Truth, cut, both_branches=False):
    """The reference's loss and dLoss at 40 digits: dict(loss, loss_floor, dloss, dloss_floor).  dloss is None where 0/0
    makes it undefined; with `both_branches` it is a list, the value with and without dLoss's cut branch (for a cut equal
    to the loss).  The floors are what float64 cannot avoid: the change a trace off by TRACE_SLACK makes, 64 units of
    roundoff of the summed magnitudes of every term, and the ground truth's rotation known only to Truth.delta (amplified by
    |invT2| / tErr in the direction of the translation error)."""
    u = mp.mpf(2) ** -52
    with mp.workdps(40):
        r = [mp.mpf(float(v)) for v in est[:3]]
        t1 = mp.matrix([mp.mpf(float(v)) for v in est[3:]])
        R1 = _rod(r)
        # loss(pose2trans(est), gt)
        T1r = R1.T
        T1t = -(R1.T * t1)
        tr = mp.fsum(truth.T[i, k] * T1r[i, k] for i in range(3) for k in range(3))
        rot_err = _rot_err(tr, PI_LOSS)
        t_err = mp.sqrt(mp.fsum((T1t[i] - truth.T[i, 3]) ** 2 for i in range(3)))
        lo = W_ROT * rot_err + W_TRANS * t_err
        lfloor = W_ROT * max(abs(_rot_err(tr + s, PI_LOSS) - rot_err) for s in (-TRACE_SLACK, TRACE_SLACK)) \
            + 64 * u * (W_ROT * rot_err + W_TRANS * (t_err + mp.fsum(abs(T1t[i]) + abs(truth.T[i, 3]) for i in range(3))))
        if lo > cut:
            lo = mp.sqrt(cut * lo)
        lo = min(lo, mp.mpf(MAXLOSS))
        # dLoss(est, trans2pose(gt))
        R2 = truth.R2
        tr = mp.fsum(R1[i, k] * R2[i, k] for i in range(3) for k in range(3))
        rot_err = _rot_err(tr, mp.pi)
        it1 = R1.T * t1
        it2 = R2.T * truth.t2
        dd = it1 - it2
        t_err = mp.sqrt(mp.fsum(x ** 2 for x in dd))
        l0 = W_ROT * rot_err + W_TRANS * t_err
        coef = _coef(tr)
        outs, floor = [], np.zeros(6)
        for cut_branch in ((True, False) if both_branches else (l0 > cut,)):
            l = mp.sqrt(l0) if cut_branch else l0
            if l > MAXLOSS or t_err + rot_err < EPS:
                outs.append(np.zeros(6))
                continue
            if t_err == 0 or coef is None:
                outs.append(None)
                continue
            g = dd / t_err
            D = _drod(r)
            scale = mp.mpf("0.5") / l if cut_branch else mp.mpf(1)
            jac, mag = [mp.mpf(0)] * 6, [mp.mpf(0)] * 6
            rel = 1 + (abs(it1[0]) + abs(it1[1]) + abs(it1[2]) + abs(it2[0]) + abs(it2[1]) + abs(it2[2])) / t_err
            for c in range(3):
                jac[3 + c] = mp.fsum(g[k] * R1[c, k] for k in range(3)) * W_TRANS
                mag[3 + c] = rel * W_TRANS
            gv = [g[k % 3] * t1[k // 3] for k in range(9)]            # g * dInvT1_dInvRot1: entry (r, r + 3c) = t[c]
            coef_moved = max(abs(c_ - coef) for c_ in (_coef(tr - TRACE_SLACK), _coef(tr + TRACE_SLACK)) if c_ is not None)
            for i in range(3):
                s_rot = mp.fsum(R2[k // 3, k % 3] * D[i, k] for k in range(9))
                jac[i] = mp.fsum(gv[k] * D[i, k] for k in range(9)) * W_TRANS + coef * s_rot * W_ROT
                mag[i] = rel * mp.fsum(abs(gv[k] * D[i, k]) for k in range(9)) * W_TRANS \
                    + abs(coef) * mp.fsum(abs(R2[k // 3, k % 3] * D[i, k]) for k in range(9)) * W_ROT
                floor[i] = max(floor[i], float(coef_moved * abs(s_rot) * W_ROT * scale))
            # a trace off by TRACE_SLACK also moves rotErr, hence the loss that dLoss's cut branch divides by
            dscale = 0
            if cut_branch:
                moved = max(abs(_rot_err(tr + s, mp.pi) - rot_err) for s in (-TRACE_SLACK, TRACE_SLACK))
                dscale = mp.mpf("0.25") * l0 ** mp.mpf("-1.5") * W_ROT * moved
            it_mag = mp.sqrt(mp.fsum(x ** 2 for x in it2))
            for i in range(6):
                floor[i] = max(floor[i], float(64 * u * mag[i] * scale)) + float(dscale * abs(jac[i])) \
                    + float(truth.delta * abs(jac[i]) * scale * (1 + it_mag / t_err))
            outs.append(np.array([float(j * scale) for j in jac]))
        return dict(loss=float(lo), loss_floor=float(lfloor), dloss=outs if both_branches else outs[0], dloss_floor=floor)


def cut_value(key, loss_at_off_cut):
    dname, dt, cut = key
    return {"off": CUT_OFF, "on": CUT_ON, "equal": float(np.float32(loss_at_off_cut))}[cut]


def classes(x):
    x = np.asarray(x, np.float64)
    return np.where(~np.isfinite(x), CLASS_NONFINITE, np.where(x == 0, CLASS_ZERO, CLASS_FINITE))


def nudged(est):
    """The estimate turned by a further 1e-8 to 3e-8 rad about each world axis: rotations float64 cannot tell from it at
    a clamped trace (trace = 3 - angle^2 + ...: 1e-8 rad moves it by about one unit in the last place)."""
    R, _ = cv2.Rodrigues(np.asarray(est[:3], np.float64).reshape(3, 1))
    out = []
    for ax in np.eye(3):
        for d in (1e-8, 2e-8, 3e-8):
            r, _ = cv2.Rodrigues(rotate(R, ax, d))
            out.append(np.concatenate([r.ravel(), est[3:]]))
    return out


def degenerate(key, loss_mp):
    """Entries whose outcome the reference's float64 arithmetic decides by rounding (see the module docstring)."""
    dname, dt, cut = key
    return dname in ("0", "1e-9", "pi") or dt == 0.0 or loss_mp >= MAXLOSS


def check_pose_loss(name, losses, dloss, pin):
    """Holds losses [N] and dloss [N, 6] of the grid around orientation `name` to the yardstick: values within 4x the float64
    oracle's distance from the 40-digit restatement plus float64's own floor and 1e-12 relative; at the degenerate entries
    the outcome class of every dLoss component must be one the compiled reference returns there.  Returns the worst
    (loss, dloss) error over the non-degenerate entries, relative to each entry's bar."""
    gt = ground_truth(name)
    truth = Truth(gt)
    gt64 = gt.astype(np.float64)
    r2, t2 = O.trans2pose(gt64)
    poses, keys = estimates(gt)
    assert np.array_equal(poses, pin[f"{name}_poses"])
    cuts, allowed = pin[f"{name}_cuts"], pin[f"{name}_class"]
    worst = [0.0, 0.0]
    n_value = 0
    for i, (est, key) in enumerate(zip(poses, keys)):
        y = yardstick(est, truth, cuts[i], both_branches=key[2] == "equal")
        lo = O.loss(O.pose2trans(est[:3], est[3:]), gt64, W_ROT, W_TRANS, cuts[i])
        bar = 4 * abs(lo - y["loss"]) + y["loss_floor"] + 1e-12 * abs(y["loss"])
        err = abs(losses[i] - y["loss"])
        assert err <= bar, (name, key, losses[i], y["loss"], lo, bar)
        worst[0] = max(worst[0], err / bar if bar > 0 else 0.0)
        cands = y["dloss"] if isinstance(y["dloss"], list) else [y["dloss"]]
        if degenerate(key, y["loss"]) or any(c is None for c in cands):
            got = classes(dloss[i])
            ok = allowed[i]
            if key[1] == 0.0:
                # the same camera centre: tErr is exactly 0 (0/0, NaN, zeros) or rounding noise (noise / noise, a finite
                # gradient in a direction of noise), depending on how two float64 products of the centre round
                ok = ok | CLASS_ZERO | CLASS_FINITE
            assert np.all(got & ok), (name, key, dloss[i], allowed[i], pin[f"{name}_dloss"][i])
            continue
        do = O.d_loss(est[:3], est[3:], r2, t2, W_ROT, W_TRANS, cuts[i]).ravel()
        best = np.inf
        for d in cands:   # a cut equal to the loss: either branch of dLoss's cut test
            b = 4 * np.abs(do - d) + y["dloss_floor"] + 1e-12 * np.abs(d)
            e = np.abs(dloss[i] - d)
            best = min(best, float(np.max(np.where(b > 0, e / np.where(b > 0, b, 1.0), np.where(e == 0, 0.0, np.inf)))))
        assert best <= 1.0, (name, key, dloss[i], cands, do, y["dloss_floor"])
        worst[1] = max(worst[1], best)
        n_value += 1
    assert n_value >= 48   # 7 of the 11 rotation distances x 3 non-zero translations, less the MAXLOSS exits
    return worst
