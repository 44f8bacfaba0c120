"""Crafted minimal sets for the sampling stage's verdicts (tests/test_host_minimal_sets.py, tests/test_gpu_minimal_sets.py).

Random draws from make_scene's smooth maps almost never give an ill-conditioned P3P, yet the sampling stage must keep the
same try as the reference on every set: its float prefilter (esac_p3p_fast.cuh) may only reject tries the exact fp64 path
rejects.  The families below aim at where a float P3P goes wrong.  Every try starts from four cells, so it can be injected
as it is: cell (cx, cy) is pixel (cx * sub + sub / 2, cy * sub + sub / 2) (no shift).  The 3D points are placed along
those rays in the camera frame, then moved to a world frame by a random rigid motion.

  cylinder   the camera centre at (1 + delta) R from the axis of the circumcircle of the first three points (R its
             radius), |delta| log-uniform in [1e-7, 1e-1], either sign: the danger cylinder, where P3P has a double root
  needle     shortest / longest squared side of the first triangle just above kPrefilterNeedle (0.02)
  parallel   two bearings with a cosine just below the 0.9999 latch: adjacent cells at f = 525, or 6 cells apart at f = 3000
  flat       the first three points almost collinear: sin^2 of the angle at point 0 just above the 1e-6 latch on det
  spread     depths of one set spread over 1e-3 .. 1e3
  noise      generic sets
Every try puts its 4th point so that the true pose misses it by e, spread over [0, 1.2 tau), and the first three points
off their rays by 0, 0.3 or 2 px (a 3D offset: the pixels are fixed by the cells).  variants() adds, for every try, the
same set scaled by 2^k (k in +-10, +-20, +-40), by 7000 and 1/7000, and moved by world offsets of 700 m and 1e5 m.

pack() lays tries out for esacb200_inject_cells: E planes of H x W cells, each try in a plane where its 4 cells are free,
and per plane 4 reserved cells holding a noise-free, well-conditioned anchor set.  Hypothesis h is injected with
[crafted, anchor], so its crafted try was accepted exactly when the device reports tries == 1.
Deterministic (numpy's default_rng) and numpy-only.
"""
from dataclasses import dataclass, field

import numpy as np

SUB, W, H = 8, 80, 60
PPX, PPY, TAU = 320.0, 240.0, 10.0
FAMILIES = ("cylinder", "needle", "parallel", "flat", "spread", "noise")
ANCHOR_CELLS = ((2, 3), (75, 4), (5, 55), (72, 52))
SCALES = tuple(2.0 ** k for k in (-40, -20, -10, 10, 20, 40)) + (7000.0, 1 / 7000.0)
OFFSETS = (700.0, 1e5)
F32_TINY, F32_MAX = float(np.finfo(np.float32).tiny), float(np.finfo(np.float32).max)


@dataclass
class Try:
    family: str
    f: float
    cells: np.ndarray                 # [4, 2] int32 (x, y)
    obj: np.ndarray                   # [4, 3] float32, world frame
    params: dict = field(default_factory=dict)

    def img(self) -> np.ndarray:
        return (self.cells * SUB + SUB // 2).astype(np.float32)


def _ray(cell, f, off=(0.0, 0.0)):
    """Direction (x/z, y/z, 1) through the pixel of `cell` moved by `off` px."""
    u = cell[0] * SUB + SUB // 2 + off[0]
    v = cell[1] * SUB + SUB // 2 + off[1]
    return np.array([(u - PPX) / f, (v - PPY) / f, 1.0])


def _off(rng, px):
    a = rng.uniform(0, 2 * np.pi)
    return (px * np.cos(a), px * np.sin(a))


def _cells(rng, n=4):
    while True:
        c = np.stack([rng.integers(0, W - 1, n), rng.integers(0, H - 1, n)], 1)
        if len({tuple(x) for x in c}) == n and not {tuple(x) for x in c} & set(ANCHOR_CELLS):
            return c.astype(np.int32)


def _solve_depth(fn, lo=0.05, hi=500.0, n=160, rng=None, vec=None):
    """A z with fn(z) = 0 in a bracket of a log grid (a random one of the brackets), or None.  vec: fn over an array."""
    zs = np.geomspace(lo, hi, n)
    v = np.array([fn(z) for z in zs]) if vec is None else vec(zs)
    idx = np.nonzero(np.isfinite(v[:-1]) & np.isfinite(v[1:]) & (np.sign(v[:-1]) != np.sign(v[1:])))[0]
    if len(idx) == 0:
        return None
    i = idx[rng.integers(len(idx))] if rng is not None else idx[0]
    a, b = zs[i], zs[i + 1]
    fa = fn(a)
    for _ in range(200):  # bisection to double precision
        m = 0.5 * (a + b)
        fm = fn(m)
        if np.sign(fm) == np.sign(fa):
            a, fa = m, fm
        else:
            b = m
        if b - a <= 1e-15 * b:
            break
    return 0.5 * (a + b)


def circumaxis_ratio(P0, P1, P2):
    """Distance of the origin from the axis of the circumcircle of P0 P1 P2, over the circle's radius (P2 may be a stack)."""
    a, b = P1 - P0, P2 - P0
    n = np.cross(a, b)
    nn = np.sum(n * n, -1)[..., None]
    c = P0 + (np.cross(n, a) * np.sum(b * b, -1)[..., None] + np.cross(b, n) * (a @ a)) / (2 * nn)  # circumcentre
    R = np.linalg.norm(c - P0, axis=-1)
    d = -c
    d = d - np.sum(d * n, -1)[..., None] / nn * n
    return np.linalg.norm(d, axis=-1) / R


def _world(rng, Pc):
    """Camera-frame points -> world frame of a random camera pose (world->camera R, t)."""
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    t = rng.uniform(-2, 2, 3)
    return ((Pc - t) @ R).astype(np.float32)  # R^T (Pc - t)


def _one(rng, family, f):
    """One try of `family` (None when this draw has no solution: the caller draws again)."""
    noise = float(rng.choice([0.0, 0.3, 2.0]))
    e4 = float(rng.uniform(0, 1.2 * TAU))
    cells = _cells(rng)
    par = {"noise_px": noise, "err4_px": e4}
    if family == "parallel":
        if f == 525.0:   # an adjacent cell: 8 px at f = 525
            d = (1, 0) if rng.integers(2) else (0, 1)
        else:            # 6 cells = 48 px at f = 3000
            d = (6, 0) if rng.integers(2) else (0, 6)
        c1 = np.minimum(cells[0] + np.array(d), [W - 2, H - 2])
        if any(tuple(c1) == tuple(c) for c in (cells[0], cells[2], cells[3])) or tuple(c1) in ANCHOR_CELLS:
            return None
        cells[1] = c1
    if family == "flat":  # three cells on one row (the third possibly one row off), point 0 between the others
        y = int(rng.integers(1, H - 2))
        xs = np.sort(rng.choice(np.arange(0, W - 1), 3, replace=False))
        cells[:3] = [[xs[1], y], [xs[0], y], [xs[2], y + int(rng.integers(0, 2))]]
        if len({tuple(c) for c in cells}) < 4 or {tuple(c) for c in cells} & set(ANCHOR_CELLS):
            return None
    dirs = [_ray(cells[i], f, _off(rng, noise)) for i in range(3)] + [_ray(cells[3], f, _off(rng, e4))]
    if family == "spread":
        z = 3.0 * 10.0 ** rng.uniform(-1.5, 1.5, 4)
        par["depth_ratio"] = float(z.max() / z.min())
    elif family == "cylinder":  # the double root is hardest on uneven depths
        z = 10.0 ** rng.uniform(0, 1.5, 4)
    else:
        z = rng.uniform(2.0, 8.0, 4)
    P = np.array([z[i] * dirs[i] for i in range(4)])

    z2 = None
    if family == "cylinder":
        delta = float(10.0 ** rng.uniform(-7, -1) * rng.choice([-1.0, 1.0]))
        par["delta"] = delta
        z2 = _solve_depth(lambda v: circumaxis_ratio(P[0], P[1], v * dirs[2]) - (1.0 + delta), rng=rng,
                          vec=lambda v: circumaxis_ratio(P[0], P[1], v[:, None] * dirs[2]) - (1.0 + delta))
    elif family == "needle":
        target = 0.02 * (1.0 + 10.0 ** rng.uniform(-4, 0))
        par["ratio"] = target

        def g(v):  # v: a depth or an array of depths
            P2 = np.multiply.outer(v, dirs[2])
            s = np.stack(np.broadcast_arrays(np.sum((P[1] - P[0]) ** 2), np.sum((P2 - P[0]) ** 2, -1), np.sum((P2 - P[1]) ** 2, -1)))
            return s.min(0) / s.max(0) - target
        z2 = _solve_depth(g, rng=rng, vec=g)
    elif family == "flat":
        target = 1e-6 * (1.0 + 10.0 ** rng.uniform(-3, 1))
        par["sin2"] = target

        def g(v):  # v: a depth or an array of depths
            a, b = P[1] - P[0], np.multiply.outer(v, dirs[2]) - P[0]
            return 1.0 - (b @ a) ** 2 / ((a @ a) * np.sum(b * b, -1)) - target
        z2 = _solve_depth(g, rng=rng, vec=g)
    if family in ("cylinder", "needle", "flat"):
        if z2 is None:
            return None
        P[2] = z2 * dirs[2]
    return Try(family, f, cells, _world(rng, P), par)


def generate(family: str, n: int, seed: int = 0, f: float = 525.0) -> list:
    rng = np.random.default_rng([seed, FAMILIES.index(family), int(f)])
    out = []
    while len(out) < n:
        t = _one(rng, family, f)
        if t is not None and np.all(np.isfinite(t.obj)):
            out.append(t)
    return out


def _normal(a) -> bool:
    m = np.abs(a.astype(np.float64))
    return bool(np.all((m >= F32_TINY) & (m * m >= F32_TINY) & (m * m <= F32_MAX)))


def variants(tries) -> list:
    """Each try scaled (SCALES) and offset (OFFSETS) in the world frame; the image side is unchanged.  Scaled copies whose
    float32 coordinates or their squares would leave the normal range are skipped."""
    out = []
    for t in tries:
        for s in SCALES:
            o = (t.obj.astype(np.float64) * s).astype(np.float32)
            if _normal(o):
                out.append(Try(t.family, t.f, t.cells, o, dict(t.params, scale=s)))
        for off in OFFSETS:
            o = (t.obj.astype(np.float64) + off).astype(np.float32)
            out.append(Try(t.family, t.f, t.cells, o, dict(t.params, offset=off)))
    return out


def anchor_obj(f: float) -> np.ndarray:
    """The anchor set: noise-free points at depths 3..4.5 on the anchor cells' rays (camera frame = world frame)."""
    return np.array([z * _ray(c, f) for z, c in zip((3.0, 3.5, 4.0, 4.5), ANCHOR_CELLS)], np.float32)


@dataclass
class Packed:
    coords: np.ndarray    # [E, 3, H, W] float32
    assign: np.ndarray    # [M] int64
    cells: np.ndarray     # [M, 2, 4, 2] int32: [crafted, anchor]
    tries: list           # the M crafted tries, in hypothesis order


def pack(tries, E: int, f: float) -> Packed:
    """First fit of every try into a plane where its 4 cells are free; tries that fit nowhere are left out."""
    coords = np.zeros((E, 3, H, W), np.float32)
    used = np.zeros((E, H, W), bool)
    anc = anchor_obj(f)
    for j, (x, y) in enumerate(ANCHOR_CELLS):
        coords[:, :, y, x] = anc[j]
        used[:, y, x] = True
    assign, cells, placed = [], [], []
    anchor_cells = np.array(ANCHOR_CELLS, np.int32)
    e = 0
    for t in tries:
        xs, ys = t.cells[:, 0], t.cells[:, 1]
        for k in range(E):
            p = (e + k) % E
            if not used[p, ys, xs].any():
                used[p, ys, xs] = True
                coords[p, :, ys, xs] = t.obj
                assign.append(p)
                cells.append(np.stack([t.cells, anchor_cells]))
                placed.append(t)
                e = (p + 1) % E
                break
    return Packed(coords, np.array(assign, np.int64), np.array(cells, np.int32).reshape(-1, 2, 4, 2), placed)


# ---- the 40-digit arbiter of a verdict that differs from cv2's --------------------------------------------------------
def root_errors(lib, obj, img, f, dps: int = 40) -> list:
    """4th-point errors (px) of every positive P3P root of the first three points, solved to `dps` digits.  Seeds: cv2's
    solveP3P and the library's fp64 p3p_solve; each is polished by Newton on the three distance equations in mpmath."""
    import cv2
    import mpmath as mp
    from oracle import esac_oracle as O
    mp.mp.dps = dps
    K = O.cam_mat(f, PPX, PPY)
    o64, i64 = obj.astype(np.float64), img.astype(np.float64)
    y = [mp.matrix([(mp.mpf(i64[i, 0]) - PPX) / f, (mp.mpf(i64[i, 1]) - PPY) / f, 1]) for i in range(4)]
    y = [v / mp.norm(v) for v in y]
    x = [mp.matrix([mp.mpf(v) for v in o64[i]]) for i in range(4)]
    pairs = ((0, 1), (0, 2), (1, 2))
    c = {p: (y[p[0]].T * y[p[1]])[0] for p in pairs}
    d2 = {p: mp.norm(x[p[0]] - x[p[1]]) ** 2 for p in pairs}
    seeds = []
    try:
        _, rvs, tvs = cv2.solveP3P(obj[:3].reshape(-1, 1, 3), img[:3].reshape(-1, 1, 2), K, None, flags=cv2.SOLVEPNP_P3P)
        for rv, tv in zip(rvs, tvs):
            R, _ = cv2.Rodrigues(rv)
            seeds.append(np.linalg.norm(o64[:3] @ R.T + tv.ravel(), axis=1))
    except cv2.error:
        pass
    yb = np.array([[float(v) for v in y[i]] for i in range(3)])
    Rs, ts = np.zeros(36), np.zeros(12)
    xs = np.ascontiguousarray(o64[:3])
    for s in range(lib.esacb200_host_p3p_all(yb.ctypes.data, xs.ctypes.data, Rs.ctypes.data, ts.ctypes.data)):
        seeds.append(np.linalg.norm(o64[:3] @ Rs[9 * s:9 * s + 9].reshape(3, 3).T + ts[3 * s:3 * s + 3], axis=1))
    # the 4th point in the frame of the scene triangle
    x1, x2, x3 = x[1] - x[0], x[2] - x[0], x[3] - x[0]
    n = mp.matrix([x1[1] * x2[2] - x1[2] * x2[1], x1[2] * x2[0] - x1[0] * x2[2], x1[0] * x2[1] - x1[1] * x2[0]])
    abc = mp.lu_solve(mp.matrix([[x1[i], x2[i], n[i]] for i in range(3)]), x3)
    roots, errs = [], []
    for sd in seeds:
        lam = mp.matrix([mp.mpf(float(v)) for v in sd])
        for _ in range(200):
            F = mp.matrix([lam[a] ** 2 + lam[b] ** 2 - 2 * c[(a, b)] * lam[a] * lam[b] - d2[(a, b)] for a, b in pairs])
            J = mp.matrix(3, 3)
            for r, (a, b) in enumerate(pairs):
                J[r, a] = 2 * lam[a] - 2 * c[(a, b)] * lam[b]
                J[r, b] = 2 * lam[b] - 2 * c[(a, b)] * lam[a]
            try:
                step = mp.lu_solve(J, F)
            except ZeroDivisionError:
                break
            lam -= step
            if mp.norm(step) < mp.mpf(10) ** (-dps + 5) * mp.norm(lam):
                break
        if min(lam) <= 0 or any(mp.norm(lam - r) < mp.mpf(10) ** (-dps // 2) * mp.norm(lam) for r in roots):
            continue
        roots.append(lam)
        P = [lam[i] * y[i] for i in range(3)]
        u1, u2 = P[1] - P[0], P[2] - P[0]
        m = mp.matrix([u1[1] * u2[2] - u1[2] * u2[1], u1[2] * u2[0] - u1[0] * u2[2], u1[0] * u2[1] - u1[1] * u2[0]])
        P3 = P[0] + abc[0] * u1 + abc[1] * u2 + abc[2] * m
        errs.append(float(mp.sqrt((f * P3[0] / P3[2] + PPX - i64[3, 0]) ** 2 + (f * P3[1] / P3[2] + PPY - i64[3, 1]) ** 2)))
    return errs


def rounding_tie(errs, tau: float = TAU, tol: float = 1e-4) -> bool:
    """Whether float64 may legitimately decide either way: the chosen root's true 4th-point error within tol of tau, or
    two roots' errors within tol of each other (the roots are ordered by that error)."""
    if not errs:
        return False
    e = sorted(errs)
    return abs(e[0] - tau) < tol or any(b - a < tol for a, b in zip(e, e[1:]))
