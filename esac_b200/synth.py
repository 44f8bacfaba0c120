"""Deterministic synthetic scene-coordinate maps (SURVEY.md section 8d).

There is no dataset and no network in this environment, so every test / bench input is generated
here: a ground-truth camera pose, a random depth map back-projected through that pose into scene
coordinates for the ground-truth expert, Gaussian noise, a fraction of uniform outliers, and pure
outlier planes for all other experts.  Intrinsics follow the reference's callers
(test_esac.py:145-147: principal point = image centre; setup_7scenes.py:6: f = 525).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def rodrigues(rvec: np.ndarray) -> np.ndarray:
    rvec = np.asarray(rvec, np.float64).reshape(3)
    th = np.linalg.norm(rvec)
    if th < 1e-12:
        return np.eye(3)
    k = rvec / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


@dataclass
class Scene:
    coords: np.ndarray       # f32 [E, 3, H, W]
    assign: np.ndarray       # i64 [M]
    gt_pose: np.ndarray      # f32 [4, 4] camera -> world (what gtPose / outPose hold)
    gt_expert: int
    f: float
    ppx: float
    ppy: float
    sub: int
    shiftX: int = 0
    shiftY: int = 0
    tau: float = 10.0
    alpha: float = 100.0
    beta: float = 0.5
    max_reproj: float = 100.0

    @property
    def params(self):
        """Positional tail of esac.forward (esac.cpp:68-77)."""
        return (self.shiftX, self.shiftY, self.f, self.ppx, self.ppy, self.tau, self.alpha, self.beta,
                self.max_reproj, self.sub)


def make_scene(E=1, H=60, W=80, M=64, sub=8, seed=0, outlier_frac=0.4, noise=0.02, f=525.0,
               outdoor=False, gt_mass=0.6, per_expert=False, shiftX=0, shiftY=0, world_offset=0.0,
               active_only=True, unit_scale=1.0, alpha=100.0, ppx=None, ppy=None) -> Scene:
    """One synthetic image worth of expert predictions.

    per_expert=False: ``assign`` is a multinomial draw of M hypotheses from a gating vector with
    ``gt_mass`` on the ground-truth expert (reference semantics: M hypotheses in total,
    test_esac.py:175).  per_expert=True: M hypotheses for every expert (M*E total, BASELINE.json's
    "256 hyp x E experts" wording).  Experts that receive no hypothesis keep all-zero planes when
    ``active_only`` (test_esac.py:157,183-185).  ``unit_scale`` multiplies every length (maps and ground-truth translation:
    metres -> e.g. millimetres) and ``alpha`` sets the score scale; the clamp fixtures use both
    (tests/golden/make_ref_golden.py).  ``ppx`` / ``ppy`` place the principal point (default: the image centre); the map
    is generated through that camera, so a pose estimated with another camera misses the ground truth."""
    rng = np.random.default_rng(1305 + seed)
    img_w, img_h = W * sub, H * sub
    ppx = img_w / 2.0 if ppx is None else float(ppx)
    ppy = img_h / 2.0 if ppy is None else float(ppy)
    box = 50.0 if outdoor else 2.0
    dmin, dmax = (5.0, 80.0) if outdoor else (1.0, 5.0)
    gt_e = int(rng.integers(E))
    centres = np.zeros((E, 3))
    for e in range(E):
        if outdoor:
            centres[e] = rng.uniform(-100, 100, 3) + world_offset
        else:
            centres[e] = np.array([5.0 * (e % 4), 5.0 * ((e // 4) % 4), 0.0]) + world_offset
    # ground-truth scene pose (world -> camera): rotation <= 30 deg, camera centre in the box
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = rng.uniform(0, np.pi / 6)
    R = rodrigues(axis * ang)
    C = centres[gt_e] + rng.uniform(-box / 2, box / 2, 3)
    t = -R @ C
    T_scene = np.eye(4)
    T_scene[:3, :3] = R
    T_scene[:3, 3] = t
    gt_pose = np.linalg.inv(T_scene).astype(np.float32)
    # pixel grid (esac_util.h:64-66)
    xs = np.arange(W) * sub + sub // 2 - shiftX
    ys = np.arange(H) * sub + sub // 2 - shiftY
    px, py = np.meshgrid(xs.astype(np.float64), ys.astype(np.float64))
    depth = rng.uniform(dmin, dmax, (H, W))
    cam = np.stack([(px - ppx) / f * depth, (py - ppy) / f * depth, depth], 0).reshape(3, -1)
    world = (R.T @ (cam - t[:, None])).reshape(3, H, W)
    world = world + rng.normal(0, noise, world.shape)
    coords = np.zeros((E, 3, H, W), np.float32)
    span = 4 * box
    for e in range(E):
        out = centres[e][:, None, None] + rng.uniform(-span / 2, span / 2, (3, H, W))
        if e == gt_e:
            mask = rng.uniform(size=(H, W)) < outlier_frac
            coords[e] = np.where(mask[None], out, world).astype(np.float32)
        else:
            coords[e] = out.astype(np.float32)
    if per_expert:
        assign = np.repeat(np.arange(E, dtype=np.int64), M)
    else:
        g = np.full(E, (1 - gt_mass) / max(E - 1, 1))
        g[gt_e] = gt_mass if E > 1 else 1.0
        g /= g.sum()
        assign = rng.choice(E, size=M, p=g).astype(np.int64)
    if active_only:
        hist = np.bincount(assign, minlength=E)
        coords[hist == 0] = 0.0
    if unit_scale != 1.0:
        coords = (coords * np.float32(unit_scale)).astype(np.float32)
        gt_pose = gt_pose.copy()
        gt_pose[:3, 3] *= np.float32(unit_scale)
    return Scene(coords, assign, gt_pose, gt_e, float(f), float(ppx), float(ppy), int(sub), shiftX, shiftY, alpha=float(alpha))


def pose_error(T_est: np.ndarray, T_gt: np.ndarray) -> tuple[float, float]:
    """(rotation error in degrees, translation error in the map's length unit) between two
    camera->world transforms, as test_esac.py:209-222 measures it."""
    T_est = np.asarray(T_est, np.float64)
    T_gt = np.asarray(T_gt, np.float64)
    Rd = T_gt[:3, :3] @ T_est[:3, :3].T
    # atan2 form: arccos(trace) alone cannot resolve angles below ~0.03 deg on float32 matrices
    sin = 0.5 * np.linalg.norm([Rd[2, 1] - Rd[1, 2], Rd[0, 2] - Rd[2, 0], Rd[1, 0] - Rd[0, 1]])
    cos = (np.trace(Rd) - 1) / 2
    return float(np.degrees(np.arctan2(sin, cos))), float(np.linalg.norm(T_est[:3, 3] - T_gt[:3, 3]))
