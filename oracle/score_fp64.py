"""Float64 restatement of getReproErrs (no-Jacobian path) + getHypScores for given poses (test infrastructure only).

Every step is the plain mathematical operation, evaluated in float64 on the float32 scene coordinates:
  R = Rodrigues(rvec);  X_cam = R X + t;  OpenCV's `z ? 1/z : 1` (no cheirality test);
  pixel centre = (x sub + sub//2 - shiftX, y sub + sub//2 - shiftY);
  err = min(|proj - pixel|, maxReproj), a non-finite error counts as maxReproj (the scoring kernel's rule, DESIGN.md §2);
  w = 1 - sigmoid(beta (err - tau));  score = alpha / N * sum(w).
It shares no code with the cv2 oracle (oracle/esac_oracle.py) or the C restatement (oracle/esac_oracle_c.c), so it pins the
scoring kernel to the operation rather than to another implementation's rounding.  Hypotheses are processed in chunks, so
64 poses x 480x640 cells take a few seconds."""
from __future__ import annotations

import numpy as np


def rodrigues(rvecs: np.ndarray) -> np.ndarray:
    """[M, 3] rotation vectors -> [M, 3, 3] matrices (identity below DBL_EPSILON, as cv::Rodrigues)."""
    r = np.asarray(rvecs, np.float64).reshape(-1, 3)
    th = np.linalg.norm(r, axis=1)
    small = th < np.finfo(np.float64).eps
    k = r / np.where(small, 1.0, th)[:, None]
    c, s = np.cos(th)[:, None, None], np.sin(th)[:, None, None]
    kx = np.zeros((len(r), 3, 3))
    kx[:, 0, 1], kx[:, 0, 2], kx[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    kx[:, 1, 0], kx[:, 2, 0], kx[:, 2, 1] = k[:, 2], -k[:, 1], k[:, 0]
    R = c * np.eye(3) + (1 - c) * np.einsum("mi,mj->mij", k, k) + s * kx
    R[small] = np.eye(3)
    return R


def pixel_centres(H: int, W: int, sub: int, shiftX: int, shiftY: int) -> tuple[np.ndarray, np.ndarray]:
    """Pixel centre of every cell, [H, W] each (createSampling: integer arithmetic, sub // 2)."""
    xs = np.arange(W, dtype=np.int64) * sub + sub // 2 - shiftX
    ys = np.arange(H, dtype=np.int64) * sub + sub // 2 - shiftY
    px, py = np.meshgrid(xs.astype(np.float64), ys.astype(np.float64))
    return px, py


def repro_errs(coords, assign, poses6, shiftX, shiftY, f, ppx, ppy, max_reproj, sub, chunk: int = 8) -> np.ndarray:
    """Reprojection errors [M, H, W] (float64, clamped to max_reproj) of every pose on its expert's plane."""
    coords = np.asarray(coords)
    E, _, H, W = coords.shape
    assign = np.asarray(assign, np.int64).reshape(-1)
    poses6 = np.asarray(poses6, np.float64).reshape(-1, 6)
    M = len(assign)
    px, py = pixel_centres(H, W, sub, shiftX, shiftY)
    px, py = px.reshape(-1), py.reshape(-1)
    planes = coords.reshape(E, 3, H * W).astype(np.float64)
    Rs = rodrigues(poses6[:, :3])
    out = np.empty((M, H * W))
    for h0 in range(0, M, chunk):
        hs = np.arange(h0, min(M, h0 + chunk))
        X = planes[assign[hs]]                                          # [m, 3, N]
        cam = np.einsum("mij,mjn->min", Rs[hs], X) + poses6[hs, 3:, None]
        z = cam[:, 2]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            iz = np.where(z != 0, 1.0 / np.where(z != 0, z, 1.0), 1.0)
            u = cam[:, 0] * iz * f + ppx
            v = cam[:, 1] * iz * f + ppy
            err = np.hypot(u - px, v - py)
        err = np.where(np.isfinite(err), np.minimum(err, max_reproj), max_reproj)
        out[hs] = err
    return out.reshape(M, H, W)


def soft_inlier_weights(errs, tau, beta) -> np.ndarray:
    """w = 1 - sigmoid(beta (err - tau)), computed without overflow."""
    x = beta * (np.asarray(errs, np.float64) - tau)
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, e / (1.0 + e), 1.0 / (1.0 + e))


def score(coords, assign, poses6, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, max_reproj, sub,
          chunk: int = 8) -> tuple[np.ndarray, np.ndarray]:
    """(scores [M], per-cell weights [M, H, W]) for the positional tail of esac.forward (shiftX .. subSampling)."""
    errs = repro_errs(coords, assign, poses6, shiftX, shiftY, f, ppx, ppy, max_reproj, sub, chunk)
    w = soft_inlier_weights(errs, tau, beta)
    M, H, W = w.shape
    return alpha / (H * W) * w.reshape(M, -1).sum(axis=1), w
