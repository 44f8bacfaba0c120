"""CPU ORACLE for the ESAC differentiable-RANSAC hot path (esac.forward / esac.backward).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it.  The product path (``esac_b200``) never routes through this file.

What it is: a line-by-line restatement, in Python on top of the *real* OpenCV
(``cv2`` 4.13 wheel: ``solvePnP`` P3P / ITERATIVE, ``projectPoints``, ``Rodrigues``), of the
reference's native extension

    code/esac/esac.cpp          esac_forward  64-190, esac_backward 213-511
    code/esac/esac_util.h       createSampling 53-70, safeSolvePnP 85-114,
                                                sampleHypotheses 129-225, getHypScores 235-260,
                                                getReproErrs 274-363, refineHyp 378-454,
                                                softMax 461-482, entropy 489-497, draw 505-530,
                                                pose2trans 537-548, trans2pose 555-568, getMax 599-612
    code/esac/esac_derivative.h dProjectdObj 47-102, dPNP 128-185,
                                                dScore 205-324, dSMScore 347-420
    code/esac/esac_loss.h       calcAngularDistance 45-55, loss 66-83, dLoss 94-210

including the float/double mix, the x-outer/y-inner point order, EPS / PROB_THRESH / MAXLOSS,
the ``> 10`` clamps, the dLoss cut quirk, ``PI`` vs ``CV_PI`` and the ``irand`` off-by-one
(last row / column never sampled).

PARITY PINNED against the reference's own compiled code: oracle/_ref/esac_ref is the unmodified
code/esac/{esac.cpp, thread_rand.cpp} + headers, compiled by oracle/build_ref.py against a minimal
<opencv2/opencv.hpp> stand-in whose solvePnP / projectPoints / Rodrigues / Mat::inv are executed by the real OpenCV of the
cv2 wheel.  Run single-threaded on its default std::mt19937 stream (reproduced here by ThreadRandStream) it returns the
same winning expert, a bit-identical pose, the same expected loss (<= 5e-11) and the same gradients (<= 3e-9 relative)
as this file on every case of tests/test_ref_pin.py and tests/golden/make_ref_golden.py, including 480x640 and
world-scale maps; its outputs are committed as tests/golden/ref_*.npz.  What remains unpinned: OpenCV 4.13 (the wheel)
instead of the 3.4.2 the reference's README names -- no 3.4.2 binary exists in this image.

One deliberate, documented deviation: the reference draws minimal sets from per-OpenMP-thread
``std::mt19937`` streams (thread_rand.cpp:13-30) whose consumption order depends on the OpenMP
schedule -- with more than one thread its sample stream is not reproducible even against itself.
Besides the single-thread stream (``mt=ThreadRandStream()``, used for the pin) the oracle therefore
offers the counter-based generator ``cell_draw`` below (shared, bit for bit, with the CUDA path)
and explicit minimal-set injection (``injected_cells``).  The
*distribution* is the reference's: x in [0, W-2], y in [0, H-2], 4 distinct cells, retry until
the 4-point reprojection gate passes.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import cv2
import numpy as np

# esac_util.h:39-40, esac_derivative.h:33, esac_loss.h:33, esac.cpp:44-45
EPS = 0.00000001
PI = 3.1415926
PROB_THRESH = 0.001
MAXLOSS = 10000000.0
MAX_SAMPLING_TRIES = 1000000
MAX_REF_STEPS = 100

_M64 = (1 << 64) - 1
_GOLD = 0x9E3779B97F4A7C15


# --------------------------------------------------------------------------------------
# counter-based sampling stream (shared with esac_b200/csrc/esac_rng.cuh)
# --------------------------------------------------------------------------------------
def mix64(z: int) -> int:
    z &= _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def try_state(seed: int, h: int, t: int) -> int:
    s = mix64(seed + _GOLD * (h + 1))
    return mix64(s + _GOLD * (t + 1))


def cell_draw(state: int, k: int, W: int, H: int) -> tuple[int, int]:
    """k-th (x, y) draw of a try.  x in [0, W-2], y in [0, H-2]: reproduces
    irand(0, imW-1) -> uniform_int(0, imW-2) (thread_rand.cpp:68-71, esac_util.h:167-168)."""
    r = mix64(state + _GOLD * (k + 1))
    x = ((r & 0xFFFFFFFF) * (W - 1)) >> 32
    y = ((r >> 32) * (H - 1)) >> 32
    return int(x), int(y)


def draw_minimal_set(seed: int, h: int, t: int, W: int, H: int) -> list[tuple[int, int]]:
    """4 distinct cells; duplicates are re-drawn (esac_util.h:164-176)."""
    st = try_state(seed, h, t)
    cells: list[tuple[int, int]] = []
    k = 0
    while len(cells) < 4:
        c = cell_draw(st, k, W, H)
        k += 1
        if c in cells:
            continue
        cells.append(c)
    return cells


# --------------------------------------------------------------------------------------
# the reference's own stream (thread_rand.cpp:7-71) for ONE OpenMP thread
# --------------------------------------------------------------------------------------
class ThreadRandStream:
    """std::mt19937 seeded like ThreadRand::init (thread_rand.cpp:13-30: generator i gets seed + i; default seed 1305)
    + libstdc++'s std::uniform_int_distribution<int> (GCC >= 11: Lemire's nearly-divisionless reduction of one 32-bit
    draw, bits/uniform_int_dist.h `_S_nd`).  With OMP_NUM_THREADS=1 the compiled reference consumes exactly this stream,
    hypothesis after hypothesis, try after try -- which is how tests/test_ref_pin.py runs oracle/_ref and this oracle on
    identical minimal sets.  The state persists across calls, as the reference's static generators do."""

    def __init__(self, seed: int = 1305, tid: int = 0):
        self.bg = np.random.MT19937()
        self.bg._legacy_seeding(int(seed) + int(tid))  # init_genrand(seed) == std::mt19937::seed(seed)
        self._buf = np.empty(0, np.uint64)
        self._pos = 0
        self.draws = 0

    def _next32(self) -> int:
        if self._pos >= len(self._buf):
            self._buf = self.bg.random_raw(4096)
            self._pos = 0
        v = int(self._buf[self._pos])
        self._pos += 1
        self.draws += 1
        return v

    def irand(self, inc_min: int, exc_max: int) -> int:
        """irand(incMin, excMax) -> uniform_int_distribution(incMin, excMax - 1) (thread_rand.cpp:68-71)."""
        rng = (exc_max - 1) - inc_min + 1
        p = self._next32() * rng
        low = p & 0xFFFFFFFF
        if low < rng:
            thr = ((1 << 32) - rng) % rng
            while low < thr:
                p = self._next32() * rng
                low = p & 0xFFFFFFFF
        return inc_min + (p >> 32)


def draw_minimal_set_mt(mt: ThreadRandStream, W: int, H: int) -> list[tuple[int, int]]:
    """esac_util.h:164-176 on the reference's own stream: x = irand(0, imW-1), y = irand(0, imH-1), duplicates re-drawn."""
    cells: list[tuple[int, int]] = []
    while len(cells) < 4:
        x = mt.irand(0, W - 1)
        y = mt.irand(0, H - 1)
        if (x, y) in cells:
            continue
        cells.append((x, y))
    return cells


# --------------------------------------------------------------------------------------
# hypothesis assignment of the callers (train_esac.py:130-140, test_esac.py:169-177, util.py:38-48)
# --------------------------------------------------------------------------------------
def clamp_probs(probs: np.ndarray, n: int) -> np.ndarray:
    """util.clamp_probs: all entries but the n largest become zero (n < 0: unchanged).  The reference walks the
    ascending sort order and zeroes the first len-n indices (util.py:43-48); ties are broken as a stable sort does."""
    probs = np.array(probs, np.float32, copy=True)
    if n < 0:
        return probs
    order = np.argsort(probs, kind="stable")
    for i, idx in enumerate(order):
        if i < probs.shape[0] - n:
            probs[idx] = 0
    return probs


def assign_hypotheses(weights, M: int, seed: int, keep_top: int = -1, single: bool = False):
    """e_hyps, e_hyps_hist for a batch of gating outputs [B, E]: clamp_probs, then M draws with replacement from the
    categorical distribution weights/sum(weights) (torch.multinomial semantics: any non-negative weights), then the
    histogram over experts (torch.histc with one bin per expert).  Draw h of image b inverts the fp64 running sum at
    u = uniform53(try_state(seed, b, h)) * total; `single` repeats draw 0 (expertselection, train_esac.py:133-135)."""
    weights = np.asarray(weights, np.float32)
    B, E = weights.shape
    assign = np.zeros((B, M), np.int64)
    hist = np.zeros((B, E), np.float32)
    for b in range(B):
        w = clamp_probs(weights[b], keep_top)
        if not np.all(np.isfinite(w)) or np.any(w < 0):
            raise RuntimeError("probability tensor contains either inf, nan or element < 0")
        cdf = np.zeros(E, np.float64)
        acc = 0.0
        last_pos = -1
        for e in range(E):
            if w[e] > 0:
                acc += float(w[e])
                last_pos = e
            cdf[e] = acc
        if last_pos < 0:
            raise RuntimeError("invalid multinomial distribution (sum of probabilities <= 0)")
        total = cdf[E - 1]
        for h in range(M):
            r = try_state(seed, b, 0 if single else h)
            u = float(r >> 11) * 2.0 ** -53 * total
            e = int(np.searchsorted(cdf, u, side="right"))  # first e with cdf[e] > u
            if e >= E:
                e = last_pos
            assign[b, h] = e
            hist[b, e] += 1
    return assign, hist


# --------------------------------------------------------------------------------------
# small helpers
# --------------------------------------------------------------------------------------
def cam_mat(f: float, ppx: float, ppy: float) -> np.ndarray:
    """esac.cpp:93-97: float 3x3."""
    K = np.eye(3, dtype=np.float32)
    K[0, 0] = np.float32(f)
    K[1, 1] = np.float32(f)
    K[0, 2] = np.float32(ppx)
    K[1, 2] = np.float32(ppy)
    return K


def create_sampling(W: int, H: int, sub: int, shiftX: int, shiftY: int) -> np.ndarray:
    """esac_util.h:53-70.  Returns int32 [H, W, 2] (x, y); sub/2 is integer division."""
    xs = np.arange(W, dtype=np.int64) * sub + sub // 2 - shiftX
    ys = np.arange(H, dtype=np.int64) * sub + sub // 2 - shiftY
    s = np.empty((H, W, 2), np.int32)
    s[:, :, 0] = xs[None, :]
    s[:, :, 1] = ys[:, None]
    return s


def safe_solve_pnp(obj, img, K, rvec, tvec, guess: bool, flag: int):
    """esac_util.h:85-114.  Returns (ok, rvec(3,1) f64, tvec(3,1) f64)."""
    obj = np.ascontiguousarray(obj, np.float32).reshape(-1, 1, 3)
    img = np.ascontiguousarray(img, np.float32).reshape(-1, 1, 2)
    try:
        if guess:
            ok, r, t = cv2.solvePnP(obj, img, K, None, np.array(rvec, np.float64).reshape(3, 1).copy(),
                                    np.array(tvec, np.float64).reshape(3, 1).copy(), True, flag)
        else:
            ok, r, t = cv2.solvePnP(obj, img, K, None, flags=flag)
    except cv2.error:
        ok = False
    if not ok:
        return False, np.zeros((3, 1)), np.zeros((3, 1))
    return True, np.asarray(r, np.float64).reshape(3, 1), np.asarray(t, np.float64).reshape(3, 1)


def _cell_obj(coords: np.ndarray, e: int, x: int, y: int) -> np.ndarray:
    return np.array([coords[e, 0, y, x], coords[e, 1, y, x], coords[e, 2, y, x]], np.float32)


@dataclass
class Hyp:
    rvec: np.ndarray  # (3,1) f64
    tvec: np.ndarray  # (3,1) f64
    cells: list = field(default_factory=list)  # 4 x (x, y)
    img: np.ndarray | None = None  # (4,2) f32
    obj: np.ndarray | None = None  # (4,3) f32
    tries: int = 0


# --------------------------------------------------------------------------------------
# esac_util.h
# --------------------------------------------------------------------------------------
def sample_hypotheses(coords, assign, sampling, K, max_tries, tau, seed=1305, injected_cells=None, mt=None):
    """esac_util.h:129-225.  ``injected_cells``: int array [M, T, 4, 2] of candidate minimal sets
    (x, y) per hypothesis, tried in order; ``mt``: a ThreadRandStream = the reference's own single-thread stream;
    otherwise the counter stream (seed, h, t)."""
    E, _, H, W = coords.shape
    hyps = []
    for h in range(len(assign)):
        e = int(assign[h])
        hyp = Hyp(np.zeros((3, 1)), np.zeros((3, 1)))
        n_tries = max_tries if injected_cells is None else min(max_tries, injected_cells.shape[1])
        for t in range(n_tries):
            if mt is not None:
                cells = draw_minimal_set_mt(mt, W, H)
            elif injected_cells is None:
                cells = draw_minimal_set(seed, h, t, W, H)
            else:
                cells = [(int(c[0]), int(c[1])) for c in injected_cells[h, t]]
            img = np.array([sampling[y, x] for (x, y) in cells], np.float32)  # Point2i -> Point2f
            obj = np.array([_cell_obj(coords, e, x, y) for (x, y) in cells], np.float32)
            hyp.cells, hyp.img, hyp.obj, hyp.tries = cells, img, obj, t + 1
            ok, hyp.rvec, hyp.tvec = safe_solve_pnp(obj, img, K, None, None, False, cv2.SOLVEPNP_P3P)
            if not ok:
                continue
            proj, _ = cv2.projectPoints(obj.reshape(-1, 1, 3), hyp.rvec, hyp.tvec, K, None)
            proj = proj.reshape(-1, 2).astype(np.float32)
            d = img - proj  # float
            n = np.sqrt(d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2)
            if np.all(n < tau):  # NaN compares false -> outlier -> retry
                break
        hyps.append(hyp)
    return hyps


def _collect(coords, e, sampling):
    """x-outer / y-inner correspondences (esac_util.h:292-305): point p = x*H + y."""
    H, W = sampling.shape[:2]
    pts3 = np.ascontiguousarray(coords[e].transpose(2, 1, 0).reshape(W * H, 3), np.float32)
    pts2 = np.ascontiguousarray(sampling.transpose(1, 0, 2).reshape(W * H, 2)).astype(np.float32)
    return pts3, pts2


def get_repro_errs(coords, rvec, tvec, e, sampling, K, max_reproj, calc_j=False):
    """esac_util.h:274-363.  Returns (errs f32 [H, W], jacobeanHyp f64 [N, 6] or None)."""
    H, W = sampling.shape[:2]
    pts3, pts2 = _collect(coords, e, sampling)
    jac = None
    if not calc_j:
        proj, _ = cv2.projectPoints(pts3.reshape(-1, 1, 3), rvec, tvec, K, None)
        proj = proj.reshape(-1, 2)
    else:
        proj, J = cv2.projectPoints(pts3.reshape(-1, 1, 3), rvec, tvec, K, None)
        proj = proj.reshape(-1, 2)
        J = J[:, 0:6]
        d = proj.astype(np.float32) - pts2  # float Point2f difference
        err = np.maximum(np.sqrt(d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2), EPS)
        dx = 1.0 / err * d[:, 0].astype(np.float64)
        dy = 1.0 / err * d[:, 1].astype(np.float64)
        jac = dx[:, None] * J[0::2, :] + dy[:, None] * J[1::2, :]
        jac[err > max_reproj] = 0.0
    assert proj.dtype == np.float32
    cur = pts2 - proj
    l = np.sqrt(cur[:, 0].astype(np.float64) ** 2 + cur[:, 1].astype(np.float64) ** 2).astype(np.float32)
    with np.errstate(invalid="ignore"):
        l = np.minimum(l, np.float32(max_reproj))  # std::min(l, m) = (m < l) ? m : l -> NaN stays NaN
    errs = l.reshape(W, H).T.copy()
    return errs, jac


def get_hyp_scores(repro_errs, tau, alpha, beta):
    """esac_util.h:235-260."""
    scores = []
    for err in repro_errs:
        H, W = err.shape
        st = (np.float32(beta) * (err - np.float32(tau))).astype(np.float32)  # float expression
        st = st.astype(np.float64)
        st = 1.0 / (1.0 + np.exp(-st))
        # x-outer, y-inner sequential double accumulation
        s = float(np.sum((1.0 - st).T.reshape(-1)))
        fac = np.float32(np.float32(np.float32(alpha) / np.float32(W)) / np.float32(H))
        scores.append(s * float(fac))
    return scores


def refine_hyp(coords, repro_errs, sampling, K, e, tau, max_ref_steps, max_reproj, rvec, tvec):
    """esac_util.h:378-454.  Returns (rvec, tvec, inlierMap int32 [H, W] or None, rounds)."""
    H, W = sampling.shape[:2]
    local = repro_errs.copy()
    best = 4
    inlier_map = None
    rounds = 0
    pts3_all, pts2_all = _collect(coords, e, sampling)
    for _ in range(max_ref_steps):
        mask = local < np.float32(tau)  # [H, W]
        sel = mask.T.reshape(-1)  # x-outer / y-inner
        cnt = int(sel.sum())
        if cnt <= best:
            break
        best = cnt
        flag = cv2.SOLVEPNP_ITERATIVE if cnt > 4 else cv2.SOLVEPNP_P3P
        ok, r, t = safe_solve_pnp(pts3_all[sel], pts2_all[sel], K, rvec, tvec, True, flag)
        if not ok:
            break
        rvec, tvec = r, t
        inlier_map = mask.astype(np.int32)
        rounds += 1
        local, _ = get_repro_errs(coords, rvec, tvec, e, sampling, K, max_reproj)
    return rvec, tvec, inlier_map, rounds


def softmax(scores):
    """esac_util.h:461-482."""
    s = np.asarray(scores, np.float64)
    sf = np.exp(s - s.max())
    return sf / sf.sum()


def entropy(dist):
    """esac_util.h:489-497."""
    d = np.asarray(dist, np.float64)
    d = d[d > 0]
    return float(-(d * np.log2(d)).sum())


def draw(probs, training=False):
    """esac_util.h:505-530 (training is always false on the path)."""
    assert not training
    max_prob, max_idx = -1.0, 0
    for i, p in enumerate(probs):
        if p < EPS:
            continue
        if max_prob < 0 or p > max_prob:
            max_prob, max_idx = p, i
    return int(max_idx)


def pose2trans(rvec, tvec):
    """esac_util.h:537-548."""
    R, _ = cv2.Rodrigues(np.asarray(rvec, np.float64).reshape(3, 1))
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = np.asarray(tvec).reshape(3)
    return np.linalg.inv(T)


def trans2pose(T):
    """esac_util.h:555-568."""
    Ti = np.linalg.inv(np.asarray(T, np.float64))
    rvec, _ = cv2.Rodrigues(np.ascontiguousarray(Ti[:3, :3]))
    return rvec.reshape(3, 1), Ti[:3, 3].reshape(3, 1).copy()


def get_max(m):
    """esac_util.h:599-612."""
    return float(np.max(np.abs(m))) if np.size(m) else -1.0


# --------------------------------------------------------------------------------------
# esac_loss.h
# --------------------------------------------------------------------------------------
def calc_angular_distance(T1, T2):
    """esac_loss.h:45-55 (uses PI = 3.1415926)."""
    tr = float(np.trace(T2[:3, :3] @ T1[:3, :3].T))
    tr = min(3.0, max(-1.0, tr))
    return 180 * math.acos((tr - 1.0) / 2.0) / PI


def loss(T1, T2, w_rot=1.0, w_trans=1.0, cut=100.0):
    """esac_loss.h:66-83."""
    rot_err = calc_angular_distance(T1, T2)
    t_err = float(np.linalg.norm(T1[:3, 3] - T2[:3, 3]))
    l = w_rot * rot_err + w_trans * t_err
    if l > cut:
        l = math.sqrt(cut * l)
    return min(l, MAXLOSS)


def d_loss(est_r, est_t, gt_r, gt_t, w_rot=1.0, w_trans=1.0, cut=100.0):
    """esac_loss.h:94-210, quirks included (sqrt(loss) not sqrt(cut*loss); CV_PI)."""
    rot1, dRod = cv2.Rodrigues(np.asarray(est_r, np.float64).reshape(3, 1))  # dRod 3x9
    rot2, _ = cv2.Rodrigues(np.asarray(gt_r, np.float64).reshape(3, 1))
    inv1, inv2 = rot1.T, rot2.T
    diff = rot1 @ inv2
    tr = min(3.0, max(-1.0, float(np.trace(diff))))
    rot_err = 180 * math.acos((tr - 1.0) / 2.0) / math.pi
    est_t = np.asarray(est_t, np.float64).reshape(3, 1)
    gt_t = np.asarray(gt_t, np.float64).reshape(3, 1)
    invT1 = inv1 @ est_t
    invT2 = inv2 @ gt_t
    t_err = float(np.linalg.norm(invT1 - invT2))
    jac = np.zeros((1, 6))
    l = w_rot * rot_err + w_trans * t_err
    cut_loss = False
    if l > cut:
        l = math.sqrt(l)
        cut_loss = True
    if l > MAXLOSS:
        return jac
    if (t_err + rot_err) < EPS:
        return jac
    with np.errstate(all="ignore"):
        dDist_dInvT1 = ((invT1 - invT2) / t_err).reshape(1, 3)
        jac[:, 3:6] += (dDist_dInvT1 @ inv1) * w_trans
        dInvT1_dInvRot1 = np.zeros((3, 9))
        for r in range(3):
            for c in range(3):
                dInvT1_dInvRot1[r, r + 3 * c] = est_t[c, 0]
        dRodT = dRod.T  # 9x3
        jac[:, 0:3] += (dDist_dInvT1 @ dInvT1_dInvRot1 @ dRodT) * w_trans
        dRotDiff = np.zeros((9, 9))
        for b in range(3):
            dRotDiff[3 * b:3 * b + 3, 3 * b:3 * b + 3] = inv2
        dRotDiff = dRotDiff.T
        dTrace = np.zeros((1, 9))
        dTrace[0, 0] = dTrace[0, 4] = dTrace[0, 8] = 1
        dAngle = (180 / math.pi * -1 / math.sqrt(3 - tr * tr + 2 * tr)) * (dTrace @ dRotDiff @ dRodT) \
            if (3 - tr * tr + 2 * tr) > 0 else np.full((1, 3), np.nan)
        jac[:, 0:3] += dAngle * w_rot
        if cut_loss:
            jac *= 0.5 / l
    if np.isnan(jac).any():
        return np.zeros((1, 6))
    return jac


# --------------------------------------------------------------------------------------
# esac_derivative.h
# --------------------------------------------------------------------------------------
def d_project_d_obj(pt, obj, rot, trans, K, max_reproj):
    """esac_derivative.h:47-102.  pt (2,) f32, obj (3,) f32, rot 3x3 f64, trans (3,1) f64 -> 1x3."""
    f = float(K[0, 0]); ppx = float(K[0, 2]); ppy = float(K[1, 2])
    o = rot @ np.asarray(obj, np.float64).reshape(3, 1) + np.asarray(trans, np.float64).reshape(3, 1)
    X, Y, Z = float(o[0, 0]), float(o[1, 0]), float(o[2, 0])
    if abs(Z) < EPS:
        return np.zeros((1, 3))
    px = f * X / Z + ppx
    py = f * Y / Z + ppy
    ptx, pty = float(pt[0]), float(pt[1])
    err = math.sqrt((ptx - px) * (ptx - px) + (pty - py) * (pty - py))
    if err > max_reproj:
        return np.zeros((1, 3))
    err += EPS
    out = np.zeros((1, 3))
    for c in range(3):
        pxd = f * rot[0, c] / Z - f * X / Z / Z * rot[2, c]
        pyd = f * rot[1, c] / Z - f * Y / Z / Z * rot[2, c]
        out[0, c] = 0.5 / err * (2 * (ptx - px) * -pxd + 2 * (pty - py) * -pyd)
    return out


def d_project_d_obj_batch(pts2, pts3, rot, trans, K, max_reproj):
    """Vectorised d_project_d_obj over N points (same arithmetic order)."""
    f = float(K[0, 0]); ppx = float(K[0, 2]); ppy = float(K[1, 2])
    o = pts3.astype(np.float64) @ rot.T + np.asarray(trans, np.float64).reshape(1, 3)
    X, Y, Z = o[:, 0], o[:, 1], o[:, 2]
    with np.errstate(all="ignore"):
        px = f * X / Z + ppx
        py = f * Y / Z + ppy
        ptx = pts2[:, 0].astype(np.float64); pty = pts2[:, 1].astype(np.float64)
        err = np.sqrt((ptx - px) * (ptx - px) + (pty - py) * (pty - py))
        zero = (np.abs(Z) < EPS) | (err > max_reproj)
        err = err + EPS
        out = np.zeros((len(pts3), 3))
        for c in range(3):
            pxd = f * rot[0, c] / Z - f * X / Z / Z * rot[2, c]
            pyd = f * rot[1, c] / Z - f * Y / Z / Z * rot[2, c]
            out[:, c] = 0.5 / err * (2 * (ptx - px) * -pxd + 2 * (pty - py) * -pyd)
    out[zero] = 0.0
    return out


def d_pnp(img, obj, K, eps=np.float32(0.001)):
    """esac_derivative.h:128-185: central differences through P3P on float coordinates."""
    obj = np.array(obj, np.float32).copy()
    n = len(obj)
    assert n == 4
    jac = np.zeros((6, n * 3))
    eps = np.float32(eps)
    for i in range(3):  # 4th point: derivative zero (esac_derivative.h:137-138)
        for j in range(3):
            obj[i, j] = np.float32(obj[i, j] + eps)
            ok, fr, ft = safe_solve_pnp(obj, img, K, None, None, False, cv2.SOLVEPNP_P3P)
            if not ok:
                return np.zeros((6, n * 3))
            obj[i, j] = np.float32(obj[i, j] - np.float32(2) * eps)
            ok, br, bt = safe_solve_pnp(obj, img, K, None, None, False, cv2.SOLVEPNP_P3P)
            if not ok:
                return np.zeros((6, n * 3))
            obj[i, j] = np.float32(obj[i, j] + eps)
            two_eps = float(np.float32(2) * eps)  # (2 * eps) is a float expression
            jac[0:3, i * 3 + j] = ((fr - br) / two_eps).reshape(3)
            jac[3:6, i * 3 + j] = ((ft - bt) / two_eps).reshape(3)
            if np.isnan(jac[:, i * 3 + j]).any():
                return np.zeros((6, n * 3))
    return jac


def d_sm_score(coords, assign, sampling, hyps, losses, probs, repro_errs, jacobeans, K, alpha, beta, tau, max_reproj,
               clamp_thresh=10.0, clamp_log=None, g=None, support_log=None):
    """esac_derivative.h:347-420 (dSMScore) + 205-324 (dScore).  Returns list of [N_rowmajor, 3]
    f64 (index y*W + x) per hypothesis, zeros for hypotheses below PROB_THRESH.
    ``g``: per-hypothesis upstream dL/d score_h in place of the reference's p_h (l_h - sum_j p_j l_j) (``losses`` is then
    unused); ``support_log``: a list that receives each hypothesis's dPNP support term, (4, 3) f64 per minimal-set cell
    in ``hyps[h].cells`` order (zeros below PROB_THRESH)."""
    H, W = sampling.shape[:2]
    M = len(hyps)
    probs = np.asarray(probs, np.float64)
    losses = None if losses is None else np.asarray(losses, np.float64)
    upstream = g
    out = []
    for h in range(M):
        if probs[h] < PROB_THRESH:
            out.append(np.zeros((H * W, 3)))
            if support_log is not None:
                support_log.append(np.zeros((4, 3)))
            continue
        if upstream is not None:
            g = float(upstream[h])
        else:
            # scoreOutputGradients (esac_derivative.h:372-374), sequential subtraction order
            g = probs[h] * losses[h]
            for j in range(M):
                g -= probs[h] * probs[j] * losses[j]
        e = int(assign[h])
        err = repro_errs[h]
        st = (np.float32(beta) * (err - np.float32(tau))).astype(np.float32).astype(np.float64)
        st = 1.0 / (1.0 + np.exp(-st))
        dRe = -st * (1 - st) * float(np.float32(beta)) * g  # [H, W]
        fac = np.float32(np.float32(np.float32(alpha) / np.float32(W)) / np.float32(H))
        dRe = dRe * float(fac)
        dHdO = d_pnp(hyps[h].img, hyps[h].obj, K)
        if get_max(dHdO) > clamp_thresh:  # esac_derivative.h:287, "clamping for stability"
            dHdO = np.zeros_like(dHdO)
            if clamp_log is not None:
                clamp_log.append(h)
        rot, _ = cv2.Rodrigues(hyps[h].rvec)
        pts3, pts2 = _collect(coords, e, sampling)  # p = x*H + y
        w = dRe.T.reshape(-1)  # same ordering
        dPdO = d_project_d_obj_batch(pts2, pts3, rot, hyps[h].tvec, K, max_reproj) * w[:, None]
        support = (w[:, None] * jacobeans[h]).sum(axis=0).reshape(1, 6) @ dHdO  # 1x12
        if support_log is not None:
            support_log.append(support.reshape(4, 3).copy())
        g_colmajor = dPdO  # [x*H + y, 3]
        for i, (x, y) in enumerate(hyps[h].cells):
            g_colmajor[x * H + y] += support[0, 3 * i:3 * i + 3]
        out.append(g_colmajor.reshape(W, H, 3).transpose(1, 0, 2).reshape(H * W, 3).copy())
    return out


# --------------------------------------------------------------------------------------
# esac.cpp entry points
# --------------------------------------------------------------------------------------
@dataclass
class ForwardTrace:
    hyps: list
    scores: list
    probs: np.ndarray
    entropy: float
    winner: int
    ref_rvec: np.ndarray
    ref_tvec: np.ndarray
    inlier_map: np.ndarray | None
    rounds: int


def forward(coords, assign, out_pose, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, max_reproj, sub,
            seed=1305, injected_cells=None, max_tries=MAX_SAMPLING_TRIES, trace=False, mt=None):
    """esac.cpp:64-190.  coords f32 [E,3,H,W], assign i64 [M], out_pose f32 [4,4] written in place.
    Returns the winning expert index (and a ForwardTrace when ``trace``)."""
    coords = np.asarray(coords)
    assert coords.dtype == np.float32 and coords.ndim == 4
    assign = np.asarray(assign)
    assert assign.dtype == np.int64 and assign.ndim == 1
    H, W = coords.shape[2], coords.shape[3]
    K = cam_mat(f, ppx, ppy)
    sampling = create_sampling(W, H, sub, shiftX, shiftY)
    hyps = sample_hypotheses(coords, assign, sampling, K, max_tries, tau, seed, injected_cells, mt)
    errs = [get_repro_errs(coords, hy.rvec, hy.tvec, int(assign[h]), sampling, K, max_reproj)[0]
            for h, hy in enumerate(hyps)]
    scores = get_hyp_scores(errs, tau, alpha, beta)
    probs = softmax(scores)
    ent = entropy(probs)
    w = draw(probs, False)
    r, t, imap, rounds = refine_hyp(coords, errs[w], sampling, K, int(assign[w]), tau, MAX_REF_STEPS,
                                    max_reproj, hyps[w].rvec, hyps[w].tvec)
    T = pose2trans(r, t)
    out_pose[:, :] = T.astype(np.float32)
    if trace:
        return int(assign[w]), ForwardTrace(hyps, scores, probs, ent, w, r, t, imap, rounds)
    return int(assign[w])


@dataclass
class BackwardTrace:
    hyps: list
    scores: list
    probs: np.ndarray
    ref: list
    inlier_maps: list
    losses: list
    grad_I: list                # per hypothesis: dl_h . dHyp_h [N_rowmajor, 3] (None below PROB_THRESH)
    grad_II: list               # per hypothesis: the score term, dScore plus the dPNP support on the minimal set
    clamped_jr: list = None     # hypotheses whose max|J_R| > 10 zeroed path I (esac.cpp:436-437)
    clamped_dpnp: list = None   # hypotheses whose max|dPNP| > 10 zeroed the minimal-set term (esac_derivative.h:287)
    support: list = None        # per hypothesis: the dPNP support inside grad_II, (4, 3) in hyps[h].cells order
    mult: np.ndarray = None     # per hypothesis: the multiplier of grad_I in the assembly (probs, or 1 in hypotheses_vjp)


def _refined_hypotheses(coords, assign, sampling, K, tau, alpha, beta, max_reproj, max_tries, seed, injected_cells, mt):
    """esac.cpp:244-352: the hypotheses, their reprojection errors and jacobeanHyp at the initial pose, scores, softmax, and
    the refinement of every hypothesis with p >= PROB_THRESH (the others keep their initial pose and no inlier map)."""
    hyps = sample_hypotheses(coords, assign, sampling, K, max_tries, tau, seed, injected_cells, mt)
    errs, jacs = [], []
    for h, hy in enumerate(hyps):
        e_, j_ = get_repro_errs(coords, hy.rvec, hy.tvec, int(assign[h]), sampling, K, max_reproj, True)
        errs.append(e_); jacs.append(j_)
    scores = get_hyp_scores(errs, tau, alpha, beta)
    probs = softmax(scores)
    ref, imaps = [], []
    for h, hy in enumerate(hyps):
        if probs[h] < PROB_THRESH:
            ref.append((hy.rvec.copy(), hy.tvec.copy())); imaps.append(None)
            continue
        r, t, im, _ = refine_hyp(coords, errs[h], sampling, K, int(assign[h]), tau, MAX_REF_STEPS, max_reproj,
                                 hy.rvec, hy.tvec)
        ref.append((r, t)); imaps.append(im)
    return hyps, errs, jacs, scores, probs, ref, imaps


def d_hyp_d_obj(coords, e, sampling, K, rvec, tvec, inlier_map, max_reproj, clamp_thresh=10.0):
    """esac.cpp:373-449: dHyp = d (refined pose) / d (scene coordinates) of one contributing hypothesis, 6 x 3N with column
    (y*W + x)*3 + c, through J_R = -pinv(J^T J) J^T over the final inlier set at the refined pose (rvec, tvec).  Returns
    (dHyp, clamped): J_R is zeroed when max|J_R| > clamp_thresh (esac.cpp:436-437); dHyp is None when the refinement never
    accepted a round or kept fewer than 4 inliers (the reference then has no points and dHyp stays zero)."""
    H, W = sampling.shape[:2]
    if inlier_map is None:
        return None, False
    sel = np.argwhere(inlier_map.T > 0)  # rows ordered x-outer, y-inner: (x, y)
    if len(sel) < 4:
        return None, False
    dHyp = np.zeros((6, H * W * 3))
    xs, ys = sel[:, 0], sel[:, 1]
    img = sampling[ys, xs].astype(np.float32)
    obj = np.stack([coords[e, 0, ys, xs], coords[e, 1, ys, xs], coords[e, 2, ys, xs]], 1).astype(np.float32)
    proj, J = cv2.projectPoints(obj.reshape(-1, 1, 3), rvec, tvec, K, None)
    proj = proj.reshape(-1, 2).astype(np.float32)
    J = J[:, 0:6]
    d = proj - img
    err = np.maximum(np.sqrt(d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2), EPS)
    jr = (1 / err * d[:, 0].astype(np.float64))[:, None] * J[0::2] + \
         (1 / err * d[:, 1].astype(np.float64))[:, None] * J[1::2]
    jr[err > max_reproj] = 0.0
    jtj = jr.T @ jr
    inv = cv2.invert(jtj, flags=cv2.DECOMP_SVD)[1]
    JR = -inv @ jr.T  # 6 x n
    clamped = get_max(JR) > clamp_thresh
    if clamped:
        JR = np.zeros_like(JR)
    rot, _ = cv2.Rodrigues(rvec)
    dNdO = d_project_d_obj_batch(img, obj, rot, tvec, K, max_reproj)  # n x 3
    for k in range(len(xs)):
        di = int(ys[k]) * W * 3 + int(xs[k]) * 3
        dHyp[:, di:di + 3] = JR[:, k:k + 1] @ dNdO[k:k + 1, :]
    return dHyp, clamped


def assemble(out_grads, assign, probs, mult, grad_I, grad_II):
    """esac.cpp:491-508: out_grads[e] += mult_h * grad_I[h] + grad_II[h] for every hypothesis with p >= PROB_THRESH,
    float += double, sequential in h.  out_grads f32 [E,3,H,W] is accumulated in place."""
    H, W = out_grads.shape[2], out_grads.shape[3]
    for h in range(len(assign)):
        if probs[h] < PROB_THRESH:
            continue
        e = int(assign[h])
        tot = (mult[h] * grad_I[h] + grad_II[h]).reshape(H, W, 3).transpose(2, 0, 1)
        out_grads[e] = (out_grads[e].astype(np.float64) + tot).astype(np.float32)


def backward(coords, out_grads, assign, gt_pose, w_rot, w_trans, cut, shiftX, shiftY, f, ppx, ppy, tau, alpha,
             beta, max_reproj, sub, seed=1305, injected_cells=None, max_tries=MAX_SAMPLING_TRIES, trace=False, mt=None,
             clamp_thresh=10.0):
    """esac.cpp:213-511.  out_grads f32 [E,3,H,W] is ACCUMULATED in place.  Returns expected loss.
    ``clamp_thresh`` is the reference's 10 (esac.cpp:436-437, esac_derivative.h:287); tests raise it to infinity to show what
    the gradient would be without the clamps, i.e. that a fixture really trips them."""
    coords = np.asarray(coords)
    assert coords.dtype == np.float32 and coords.ndim == 4
    assert out_grads.dtype == np.float32 and out_grads.shape == coords.shape
    assign = np.asarray(assign)
    assert assign.dtype == np.int64 and assign.ndim == 1
    H, W = coords.shape[2], coords.shape[3]
    N = H * W
    M = len(assign)
    K = cam_mat(f, ppx, ppy)
    gtT = np.asarray(gt_pose, np.float32).astype(np.float64)
    sampling = create_sampling(W, H, sub, shiftX, shiftY)
    hyps, errs, jacs, scores, probs, ref, imaps = _refined_hypotheses(coords, assign, sampling, K, tau, alpha, beta,
                                                                      max_reproj, max_tries, seed, injected_cells, mt)
    losses = []
    expected = 0.0
    for h in range(M):
        T = pose2trans(*ref[h])
        losses.append(loss(T, gtT, w_rot, w_trans, cut))
        expected += probs[h] * losses[h]
    # ---- path I (esac.cpp:373-463) -----------------------------------------------------------
    gt_r, gt_t = trans2pose(gtT)
    grad_I = [None] * M
    clamped_jr, clamped_dpnp = [], []
    for h in range(M):
        if probs[h] < PROB_THRESH:
            continue
        dHyp, clamped = d_hyp_d_obj(coords, int(assign[h]), sampling, K, ref[h][0], ref[h][1], imaps[h], max_reproj,
                                    clamp_thresh)
        if clamped:
            clamped_jr.append(h)
        if dHyp is None:  # empty inlierMap (refinement never accepted a round): cols = 0 -> no points -> dHyp stays zero
            dHyp = np.zeros((6, N * 3))
        dl = d_loss(ref[h][0], ref[h][1], gt_r, gt_t, w_rot, w_trans, cut)
        grad_I[h] = (dl @ dHyp).reshape(N, 3)
    # ---- path II (esac.cpp:472-486) ----------------------------------------------------------
    support = []
    grad_II = d_sm_score(coords, assign, sampling, hyps, losses, probs, errs, jacs, K, alpha, beta, tau, max_reproj,
                         clamp_thresh, clamped_dpnp, support_log=support)
    # ---- assembly (esac.cpp:491-508): float += double, sequential over h ----------------------
    assemble(out_grads, assign, probs, probs, grad_I, grad_II)
    if trace:
        return float(expected), BackwardTrace(hyps, scores, probs, ref, imaps, losses, grad_I, grad_II, clamped_jr, clamped_dpnp,
                                              support, probs)
    return float(expected)


def hypotheses_vjp(coords, assign, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, max_reproj, sub, seed, grad_poses,
                   grad_scores, injected_cells=None, max_tries=MAX_SAMPLING_TRIES, mt=None, clamp_thresh=10.0):
    """The vector-Jacobian product of the hypotheses node (esac_b200.api.hypotheses_forward / hypotheses_backward): the
    hypotheses backward() would draw, score and refine, with the loss replaced by upstream gradients of (scores, poses).
    grad_poses [M,6] = dL/d (rvec, tvec) of the refined poses, grad_scores [M] = dL/d score_h (None counts as zero); only
    hypotheses with p >= PROB_THRESH count.  Path I takes dl = grad_poses[h] with multiplier 1, path II takes
    g = grad_scores[h]; the assembly is backward()'s.  Returns (gradient f32 [E,3,H,W], BackwardTrace with losses None)."""
    coords = np.asarray(coords)
    assert coords.dtype == np.float32 and coords.ndim == 4
    assign = np.asarray(assign)
    assert assign.dtype == np.int64 and assign.ndim == 1
    H, W = coords.shape[2], coords.shape[3]
    N = H * W
    M = len(assign)
    grad_poses = np.zeros((M, 6)) if grad_poses is None else np.asarray(grad_poses, np.float64).reshape(M, 6)
    grad_scores = np.zeros(M) if grad_scores is None else np.asarray(grad_scores, np.float64).reshape(M)
    K = cam_mat(f, ppx, ppy)
    sampling = create_sampling(W, H, sub, shiftX, shiftY)
    hyps, errs, jacs, scores, probs, ref, imaps = _refined_hypotheses(coords, assign, sampling, K, tau, alpha, beta,
                                                                      max_reproj, max_tries, seed, injected_cells, mt)
    grad_I = [None] * M
    clamped_jr, clamped_dpnp = [], []
    for h in range(M):
        if probs[h] < PROB_THRESH:
            continue
        dHyp, clamped = d_hyp_d_obj(coords, int(assign[h]), sampling, K, ref[h][0], ref[h][1], imaps[h], max_reproj,
                                    clamp_thresh)
        if clamped:
            clamped_jr.append(h)
        if dHyp is None:
            dHyp = np.zeros((6, N * 3))
        grad_I[h] = (grad_poses[h].reshape(1, 6) @ dHyp).reshape(N, 3)
    support = []
    grad_II = d_sm_score(coords, assign, sampling, hyps, None, probs, errs, jacs, K, alpha, beta, tau, max_reproj,
                         clamp_thresh, clamped_dpnp, g=grad_scores, support_log=support)
    out = np.zeros(coords.shape, np.float32)
    mult = np.ones(M)
    assemble(out, assign, probs, mult, grad_I, grad_II)
    return out, BackwardTrace(hyps, scores, probs, ref, imaps, None, grad_I, grad_II, clamped_jr, clamped_dpnp, support, mult)
