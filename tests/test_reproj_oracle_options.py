"""The reprojection-loss oracle's clamps as arguments (oracle/reproj_loss_oracle.py: max_reproj, min_depth), on the CPU:
the torch restatement against an independent numpy closed form in float64 at values other than ref_expert.py's 100 px
and 0.1, and the float64 results of the single-cell probes that tests/test_gpu_reproj_options.py holds the kernel to.

The scene and probe builders here are that file's fixtures:
  * straddling_scene: a map whose errors straddle cut and maxReproj and whose depths straddle minDepth (cells behind the
    camera included), for any pose, camera and pad;
  * probe_image: an identity ground truth, f = 512 and power-of-two depths, so that float32 and float64 place every
    cell identically; one probe cell, every other cell beyond maxReproj (gradient exactly 0)."""
import math

import numpy as np
import pytest
import torch

from oracle.reproj_loss_oracle import reproj_errors, reproj_loss_and_grad


def random_pose(rng, reach: float = 2.0) -> np.ndarray:
    """A camera->world pose [4,4] float32: uniform rotation, translation within `reach` m."""
    q = rng.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = rng.uniform(-reach, reach, 3)
    return T.astype(np.float32)


def straddling_scene(H, W, sub, seed, cut, max_reproj, min_depth):
    """(prediction [3,H,W] float32, gt [4,4] float32, f, padx, pady, ppx, ppy): per cell an error drawn around 0..1.5 cut,
    around max_reproj, log-uniform from 0.1 px to 3 max_reproj, or far beyond (below ~0.1 px the direction of the error
    is ill-conditioned in float32, and a few such cells would decide an RMS comparison; err = 0 is a probe); a depth around min_depth (half to twice
    it), behind the camera (down to -20 min_depth: the projection divides cx*zc by min_depth there), or up to 6 m beyond
    it.  f and the principal point are exact in float32.  The camera stays within 20 min_depth of the origin (at most
    2 m), so that the float32 rounding of the world coordinates stays well below a pixel at depth min_depth."""
    rng = np.random.default_rng(seed)
    gt = random_pose(rng, min(2.0, 20 * min_depth))
    f = float(np.float32(rng.uniform(400, 600)))
    padx, pady = (int(v) for v in rng.integers(-4, 5, 2))
    ppx, ppy = W * sub / 2 + 0.5 * int(rng.integers(-8, 9)), H * sub / 2 + 0.5 * int(rng.integers(-8, 9))
    n = H * W
    kind = rng.choice(4, n, p=[0.3, 0.3, 0.25, 0.15])
    err = np.select([kind == 0, kind == 1, kind == 2],
                    [rng.uniform(0, 1.5 * cut, n), rng.uniform(0.5, 1.5, n) * max_reproj,
                     10.0 ** rng.uniform(-1, math.log10(3 * max_reproj), n)], rng.uniform(5, 50, n) * max_reproj)
    depth_kind = rng.choice(3, n, p=[0.25, 0.1, 0.65])
    z = np.select([depth_kind == 0, depth_kind == 1],
                  [rng.uniform(0.5, 2.0, n) * min_depth, -rng.uniform(0.1, 20.0, n) * min_depth], min_depth + rng.uniform(0, 6, n))
    ang = rng.uniform(0, 2 * np.pi, n)
    ys, xs = np.divmod(np.arange(n), W)
    tx = xs * sub + sub / 2 - padx + err * np.cos(ang)
    ty = ys * sub + sub / 2 - pady + err * np.sin(ang)
    zz = np.maximum(z, min_depth)              # the numerator keeps the unclamped depth, the division takes the clamped one
    cam = np.stack([(tx * zz - ppx * z) / f, (ty * zz - ppy * z) / f, z, np.ones(n)])
    world = (gt.astype(np.float64) @ cam)[:3].reshape(3, H, W)
    return world.astype(np.float32), gt, f, padx, pady, ppx, ppy


def camera_coords(pred: np.ndarray, gt: np.ndarray) -> np.ndarray:
    """Camera-frame coordinates of every cell in float64, [3, H*W]."""
    Tinv = np.linalg.inv(gt.astype(np.float64))
    return Tinv[:3, :3] @ pred.reshape(3, -1).astype(np.float64) + Tinv[:3, 3:]


# ---- single-cell probes ---------------------------------------------------------------------------------------------
F_PROBE = 512.0
PROBES = ["cut+1e-4", "cut-1e-4", "max+1e-3", "max-1e-3", "depth==min", "depth-1ulp", "depth+1ulp", "behind",
          "on_target", "nan", "overflow"]


def probe_image(H, W, sub, cell, probe, cut, max_reproj, min_depth):
    """(prediction [3,H,W] float32, ppx, ppy) for the identity ground truth, f = 512, no pad: the cell `cell` (flat index)
    is the probe, every other cell lies 2 max_reproj + 7 px right of its target at depth zb (a power of two >= 2
    min_depth).  cut, max_reproj and min_depth are the float32 values the kernel sees."""
    ppx, ppy = W * sub / 2, H * sub / 2
    zb = 2.0 ** math.ceil(math.log2(2 * min_depth))
    n = H * W
    ys, xs = np.divmod(np.arange(n), W)
    tx, ty = xs * sub + sub / 2, ys * sub + sub / 2
    dx = np.full(n, 2 * max_reproj + 7)
    z = np.full(n, zb)
    md = float(np.float32(min_depth))
    if probe.startswith(("cut", "max")):
        base = cut if probe.startswith("cut") else max_reproj
        dx[cell] = base + float(probe[3:])
    elif probe == "depth==min":
        z[cell], dx[cell] = md, 3.0
    elif probe == "depth-1ulp":
        z[cell], dx[cell] = float(np.nextafter(np.float32(md), np.float32(-np.inf))), 3.0
    elif probe == "depth+1ulp":
        z[cell], dx[cell] = float(np.nextafter(np.float32(md), np.float32(np.inf))), 3.0
    elif probe == "behind":
        z[cell], dx[cell] = -zb, 3.0
    elif probe in ("on_target", "nan"):
        dx[cell] = 0.0
    elif probe == "overflow":
        dx[cell] = 2e19                        # du^2 overflows float32
    else:
        raise ValueError(probe)
    zz = np.maximum(z, md)
    pred = np.stack([((tx + dx) * zz - ppx * z) / F_PROBE, (ty * zz - ppy * z) / F_PROBE, z]).reshape(3, H, W)
    pred = pred.astype(np.float32)
    if probe == "nan":
        pred[0].flat[cell] = np.nan
    return pred, ppx, ppy


def probe_reference(pred, sub, ppx, ppy, cut, max_reproj, min_depth):
    """float64 torch: (loss, gradient [3,H,W], unclamped error [H*W]) of a probe image."""
    H, W = pred.shape[1:]
    kw = dict(image_w=2 * ppx, image_h=2 * ppy, dtype=torch.float64, min_depth=min_depth)
    loss, g = reproj_loss_and_grad(pred, torch.eye(4), F_PROBE, 0, 0, cut, sub, max_reproj=max_reproj, **kw)
    err = reproj_errors(torch.from_numpy(pred), torch.eye(4), F_PROBE, 0, 0, sub, max_reproj=math.inf, **kw)
    return loss, g.numpy(), err.numpy()


PROBE_OPTIONS = [(10.0, 100.0, 0.1), (10.0, 30.0, 1.0), (10.0, 250.0, 2.5), (10.0, 5.0, 0.01)]


def f32(*v):
    return tuple(float(np.float32(x)) for x in v)


@pytest.mark.parametrize("cut,max_reproj,min_depth", PROBE_OPTIONS)
def test_probe_cells_land_where_they_are_meant_to(cut, max_reproj, min_depth):
    """float64 places every probe on its side of its kink, the other cells beyond max_reproj with gradient exactly 0;
    the NaN cell gets a NaN gradient and the overflowing one (beyond float32, not float64) an exactly zero gradient."""
    cut, max_reproj, min_depth = f32(cut, max_reproj, min_depth)
    H, W, sub, cell = 7, 11, 8, 30
    for probe in PROBES:
        pred, ppx, ppy = probe_image(H, W, sub, cell, probe, cut, max_reproj, min_depth)
        loss, g, err = probe_reference(pred, sub, ppx, ppy, cut, max_reproj, min_depth)
        others = np.ones(H * W, bool)
        others[cell] = False
        assert (err[others] > max_reproj).all() and (g.reshape(3, -1)[:, others] == 0).all(), probe
        e, gc = err[cell], g.reshape(3, -1)[:, cell]
        zc = float(pred[2].flat[cell])
        expect = {"cut+1e-4": e > cut, "cut-1e-4": e < cut, "max+1e-3": e > max_reproj and (gc == 0).all(),
                  "max-1e-3": e < max_reproj and (gc != 0).any(), "depth==min": zc == min_depth,
                  "depth-1ulp": zc < min_depth, "depth+1ulp": zc > min_depth, "behind": zc < 0,
                  "on_target": e == 0 and (gc == 0).all(), "nan": np.isnan(gc).all(),
                  "overflow": (gc == 0).all() and e * e > np.finfo(np.float32).max}[probe]
        assert expect, (probe, e, gc, zc)
        assert math.isfinite(loss), probe


@pytest.mark.parametrize("sub,max_reproj,min_depth", [(3, 30.0, 1.0), (4, 5.0, 2.5), (1, 250.0, 0.01)])
def test_oracle_clamps_match_closed_form(sub, max_reproj, min_depth):
    """reproj_loss_and_grad(max_reproj=, min_depth=) against a closed form of ref_expert.py:103-148 with those clamps, in
    float64, on a scene whose errors and depths straddle them."""
    cut = 10.0
    pred, gt, f, padx, pady, ppx, ppy = straddling_scene(10, 13, sub, 31 + sub, cut, max_reproj, min_depth)
    X = pred.astype(np.float64)
    loss, g = reproj_loss_and_grad(torch.from_numpy(X), torch.from_numpy(gt.astype(np.float64)), f, padx, pady, cut, sub,
                                   image_w=2 * ppx, image_h=2 * ppy, dtype=torch.float64, max_reproj=max_reproj,
                                   min_depth=min_depth)
    Tinv = np.linalg.inv(gt.astype(np.float64))[:3]
    H, W = X.shape[1:]
    total = 0.0
    G = np.zeros_like(X)
    branches = set()
    for y in range(H):
        for x in range(W):
            c = Tinv[:, :3] @ X[:, y, x] + Tinv[:, 3]
            nu, nv = f * c[0] + ppx * c[2], f * c[1] + ppy * c[2]
            open_ = c[2] >= min_depth
            z = c[2] if open_ else min_depth
            du, dv = nu / z - (x * sub + sub / 2 - padx), nv / z - (y * sub + sub / 2 - pady)
            err = np.hypot(du, dv)
            e = min(err, max_reproj)
            total += e if e <= cut else np.sqrt(cut * e)
            gl = 0.0 if err > max_reproj else (1.0 if e <= cut else 0.5 * cut / np.sqrt(cut * e))
            branches.add((open_, err > max_reproj, e <= cut))
            gu, gv = gl * du / err, gl * dv / err
            gc = np.array([gu * f / z, gv * f / z, (gu * ppx + gv * ppy) / z - ((gu * nu + gv * nv) / z ** 2 if open_ else 0.0)])
            G[:, y, x] = Tinv[:, :3].T @ gc / (H * W)
    assert {b[0] for b in branches} == {True, False} and {b[1] for b in branches} == {True, False}
    # cells behind the camera divide f*xc + ppx*zc by min_depth: ~1e4 px terms cancelling to the error, hence 1e-9
    assert abs(loss - total / (H * W)) < 1e-12 * max(1.0, abs(loss))
    assert np.abs(g.numpy() - G).max() < 1e-9 * max(1.0, np.abs(G).max())
    # the defaults are ref_expert.py's literals
    l_def, g_def = reproj_loss_and_grad(X, gt.astype(np.float64), f, padx, pady, cut, sub, 2 * ppx, 2 * ppy, torch.float64)
    l_lit, g_lit = reproj_loss_and_grad(X, gt.astype(np.float64), f, padx, pady, cut, sub, 2 * ppx, 2 * ppy, torch.float64,
                                        100.0, 0.1)
    assert l_def == l_lit and torch.equal(g_def, g_lit)
