"""Oracle for the test-time evaluation (test_esac.py:209-289).  TEST INFRASTRUCTURE ONLY.

A float64 numpy restatement of what esac_b200/csrc/eval.cu computes per image, on the same algorithm: the general affine
inverse (adjugate over determinant), the nearest rotation by eight Newton steps X <- (X + X^-T) / 2 (OpenCV takes U V^T of
an SVD), and OpenCV's Rodrigues branch structure, with its exact zero where s < 1e-5 and c > 0.  The table is the
reference's loop in plain Python: per-scene lists, sorted, the upper median, strict thresholds.

A record is the 14 float64 values of esac_b200.api.EVAL_FIELDS:
rot_deg, trans_cm, correct, scene, expert, status, active, qw, qx, qy, qz, tx, ty, tz.

Only tests/ may import this module; the product path never does.
"""
from __future__ import annotations

import math

import numpy as np


def adj3(A: np.ndarray) -> np.ndarray:
    """Adjugate of a row-major 3x3 given as 9 values (esac_geom.cuh's adj3)."""
    return np.array([A[4] * A[8] - A[5] * A[7], A[2] * A[7] - A[1] * A[8], A[1] * A[5] - A[2] * A[4],
                     A[5] * A[6] - A[3] * A[8], A[0] * A[8] - A[2] * A[6], A[2] * A[3] - A[0] * A[5],
                     A[3] * A[7] - A[4] * A[6], A[1] * A[6] - A[0] * A[7], A[0] * A[4] - A[1] * A[3]])


def polar_newton(X: np.ndarray) -> np.ndarray:
    """The nearest rotation of a 3x3 (9 values): eight Newton steps, stopping at a singular matrix."""
    X = np.array(X, np.float64).reshape(9)
    for _ in range(8):
        C = adj3(X)
        dd = X[0] * C[0] + X[1] * C[3] + X[2] * C[6]
        if not abs(dd) > 0:
            break
        X = np.array([0.5 * (X[r * 3 + c] + C[c * 3 + r] / dd) for r in range(3) for c in range(3)])
    return X


def affine_inverse(T: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(rotation block, translation) of the inverse of an affine 4x4 (16 values, last row 0 0 0 1)."""
    T = np.asarray(T, np.float64).reshape(16)
    R = T[[0, 1, 2, 4, 5, 6, 8, 9, 10]]
    B = adj3(R)
    d = R[0] * B[0] + R[1] * B[3] + R[2] * B[6]
    Ri = B / d
    t = np.array([-(Ri[r * 3] * T[3] + Ri[r * 3 + 1] * T[7] + Ri[r * 3 + 2] * T[11]) for r in range(3)])
    return Ri, t


def rodrigues_sin_cos(R: np.ndarray) -> tuple[np.ndarray, float, float]:
    """The skew part, s and clamped c that OpenCV's Rodrigues branches on."""
    v = np.array([R[7] - R[5], R[2] - R[6], R[3] - R[1]])
    s = math.sqrt((v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) * 0.25)
    c = min(max((R[0] + R[4] + R[8] - 1) * 0.5, -1.0), 1.0)
    return v, s, c


def rodrigues_m2v(R: np.ndarray) -> np.ndarray:
    """Rotation matrix (9 values) -> axis-angle vector, OpenCV's branches (esac_geom.cuh's rodrigues_m2v)."""
    v, s, c = rodrigues_sin_cos(R)
    theta = math.acos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        rx = math.sqrt(max((R[0] + 1) * 0.5, 0.0))
        ry = math.sqrt(max((R[4] + 1) * 0.5, 0.0)) * (-1.0 if R[1] < 0 else 1.0)
        rz = math.sqrt(max((R[8] + 1) * 0.5, 0.0)) * (-1.0 if R[2] < 0 else 1.0)
        if abs(rx) < abs(ry) and abs(rx) < abs(rz) and ((R[5] > 0) != (ry * rz > 0)):
            rz = -rz
        theta /= math.sqrt(rx * rx + ry * ry + rz * rz)
        return np.array([rx, ry, rz]) * theta
    return v * (1 / (2 * s) * theta)


def rotation_error_deg(out_pose: np.ndarray, gt_pose: np.ndarray) -> float:
    """|Rodrigues(P_R G_R^T)| in degrees, 0 in OpenCV's s < 1e-5, c > 0 branch."""
    P = np.asarray(out_pose, np.float64).reshape(4, 4)
    G = np.asarray(gt_pose, np.float64).reshape(4, 4)
    X = polar_newton((P[:3, :3] @ G[:3, :3].T).reshape(9))
    _, s, c = rodrigues_sin_cos(X)
    return 0.0 if (s < 1e-5 and c > 0) else math.acos(c) * 180.0 / math.pi


def pose_file_entry(out_pose: np.ndarray) -> np.ndarray:
    """qw qx qy qz tx ty tz of test_esac.py:231-247 (q_xyz NaN at angle 0, as there)."""
    Ri, t = affine_inverse(out_pose)
    r = rodrigues_m2v(polar_newton(Ri))
    angle = math.sqrt(float(r @ r))
    with np.errstate(invalid="ignore", divide="ignore"):
        axis = r / angle
    return np.concatenate([[math.cos(angle * 0.5)], math.sin(angle * 0.5) * axis, t])


def evaluate(out_pose, gt_pose, expert: int, scene: int, hist=None, status: int = 0) -> np.ndarray:
    """One image's record (float64 [14])."""
    P = np.asarray(out_pose, np.float64).reshape(4, 4)
    G = np.asarray(gt_pose, np.float64).reshape(4, 4)
    trans_cm = math.sqrt(float(((G[:3, 3] - P[:3, 3]) ** 2).sum())) * 100.0
    active = float(np.count_nonzero(np.asarray(hist) > 0)) if hist is not None else math.nan
    head = [rotation_error_deg(P, G), trans_cm, float(int(expert) == int(scene)), float(scene), float(expert), float(status),
            active]
    return np.concatenate([head, pose_file_entry(P)])


def evaluate_batch(out_poses, gt_poses, experts, scenes, hist=None, status=None) -> np.ndarray:
    """Records [B,14] of a batch."""
    B = len(out_poses)
    return np.stack([evaluate(out_poses[b], gt_poses[b], experts[b], scenes[b], None if hist is None else hist[b],
                              0 if status is None else int(status[b])) for b in range(B)])


def table(records, num_scenes: int, rot_threshold: float = 5.0, trans_threshold: float = 5.0, average: bool = True) -> dict:
    """test_esac.py:249-289 over the counted records (status 0, scene in [0, num_scenes)): the console lines, the
    results-file lines and the experts-active lines, plus the number of records left out."""
    scenes_r = [[] for _ in range(num_scenes)]
    scenes_t = [[] for _ in range(num_scenes)]
    scenes_c = [[] for _ in range(num_scenes)]
    avg_active, max_active, images, excluded = 0.0, 0.0, 0, 0
    for rec in np.asarray(records, np.float64).reshape(-1, 14):
        scene = int(rec[3])
        if rec[5] != 0 or not 0 <= scene < num_scenes:
            excluded += 1
            continue
        images += 1
        scenes_r[scene].append(float(rec[0]))
        scenes_t[scene].append(float(rec[1]))
        scenes_c[scene].append(rec[2] == 1.0)
        avg_active += float(rec[6])
        max_active = max(max_active, float(rec[6]))
    console = ["Scene - Class.Acc. - Pose.Acc. - Median Rot. - Median Trans.",
               "------------------------------------------------------------"]
    results = []
    avg_class = avg_pose = avg_rot = avg_trans = 0

    def median(l):
        if len(l) == 0:
            return 0
        l.sort()
        return l[int(len(l) / 2)]

    for sceneIdx in range(num_scenes):
        class_acc = sum(scenes_c[sceneIdx]) / max(len(scenes_c[sceneIdx]), 1)
        avg_class += class_acc
        pose_acc = [(t_err < trans_threshold and r_err < rot_threshold)
                    for (t_err, r_err) in zip(scenes_t[sceneIdx], scenes_r[sceneIdx])]
        pose_acc = sum(pose_acc) / max(len(pose_acc), 1)
        avg_pose += pose_acc
        median_r = median(scenes_r[sceneIdx])
        avg_rot += median_r
        median_t = median(scenes_t[sceneIdx])
        avg_trans += median_t
        console.append("%7d %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (sceneIdx, class_acc * 100, pose_acc * 100, median_r,
                                                                    median_t))
        results.append("%f %f %f %f" % (class_acc, pose_acc, median_r, median_t))
    if average:
        console.append("------------------------------------------------------------")
        console.append("Average %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (
            avg_class * 100 / num_scenes, avg_pose * 100 / num_scenes, avg_rot / num_scenes, avg_trans / num_scenes))
    n = max(images, 1)
    experts = [f"Avg. experts active: {avg_active / n}", f"Max. experts active: {max_active}"]
    return {"console": console, "results": results, "experts": experts, "excluded": excluded}


def pose_line(name: str, rec) -> str:
    """One pose-file line (test_esac.py:244-247); `name` is the already stripped file name."""
    return "%s %f %f %f %f %f %f %f" % (name, *(float(v) for v in np.asarray(rec)[7:14]))
