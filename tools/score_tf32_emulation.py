"""CPU emulation of the scoring kernel's per-cell arithmetic (score.cu) under candidate changes, against the float64
reference (oracle/score_fp64.py) on the single-cell probe maps and dense scenes of tests/test_gpu_score_shapes.py.

Transform (xc, yc, zc) = A (X, Y, Z) + b, rows folded in fp64 and rounded to fp32 as fold_kernel does:
  fp32     today's kernel: three dependent FFMAs per component;
  3xtf32   tensor-core form, v = big + small with big = cvt.rna.tf32(v), small = cvt.rna.tf32(v - big):
           m16n8k8 [a_big, b_big, a_big, b_small] . [X_big, 1, X_small, 1], then m16n8k4 [a_small, 0] . [X_big, 1]
           accumulated onto it (CUTLASS's 3xTF32: no small x small term);
  4xtf32   3xtf32 plus the small x small term (second MMA K = 8).
Accumulation of an MMA: `nearest` adds the exact TF32 products exactly and rounds once; `trunc` aligns every term to the
largest exponent, truncates it to 24 bits, and truncates the sum to fp32 (what published measurements of earlier tensor
cores report).  `fold` scales the rows that carry f and the principal-point offsets by k1 = beta log2(e) and takes one
reciprocal per pair of cells, w_a + w_b = 2^-32 (d_a + d_b) / (d_a d_b) with d = 2^-32 + 2^(t - 32).  MUFU results are
taken as correctly rounded.

Prints, per variant, the largest error of a cell pair's summed weight over every pair of the probe maps (the GPU probes
hold one cell's weight to 1e-5; the other cell of a probe's pair weighs ~e^-45) and the largest |score - float64 score| of the dense scenes (held to 1e-4).

    python tools/score_tf32_emulation.py [--maps 480x640,120x160]
"""
import argparse
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import numpy as np  # noqa: E402

from esac_b200.synth import make_scene  # noqa: E402
from oracle import score_fp64  # noqa: E402
from test_gpu_score_shapes import DENSE, PROBE_SHAPES, _dense_poses, probe_scene  # noqa: E402

F32, F64 = np.float32, np.float64
LOG2E = F32(1.4426950408889634)
SHIFT = 32


def tf32_rna(v):
    """cvt.rna.tf32.f32 of finite values: 10 explicit mantissa bits, ties away from zero."""
    b = np.asarray(v, F32).view(np.uint32).astype(np.uint64)
    return ((b + 0x1000) & 0xFFFFE000).astype(np.uint32).view(F32)


def _trunc(v, e):
    q = np.exp2(e - 23)
    return np.trunc(v / q) * q


def mma(terms, c, trunc):
    allv = np.concatenate([np.stack(terms), c[None]], 0).astype(F64)
    if not trunc:
        return allv.sum(0).astype(F32)
    big = np.abs(allv).max(0)
    s = _trunc(allv, np.floor(np.log2(np.where(big > 0, big, 1.0)))).sum(0)
    return _trunc(s, np.floor(np.log2(np.where(s != 0, np.abs(s), 1.0)))).astype(F32)


def fma(a, b, c):
    return (F64(a) * F64(b) + F64(c)).astype(F32)


def plane_centre(plane):
    """prep_kernel's strided-sample mean."""
    N = plane.shape[1]
    ns = min(N, 4096)
    idx = np.minimum(np.arange(ns) * max(1, N // ns), N - 1)
    return plane[:, idx].astype(F64).mean(1).astype(F32)


def weights(coords, assign, poses6, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, max_reproj, sub, transform="fp32",
            trunc=False, fold=False):
    """Per-cell weights [M, N] as the variant computes them; with `fold` each pair's sum is split evenly over its cells
    (compare pair sums, or scores, only)."""
    E, _, H, W = coords.shape
    N = H * W
    planes = coords.reshape(E, 3, N)
    px, py = score_fp64.pixel_centres(H, W, sub, shiftX, shiftY)
    k1 = F32(beta) * LOG2E
    k0 = -F32(beta) * F32(tau) * LOG2E
    kf = k1 if fold else F32(1)
    aa = (kf * (F32(ppx) - px.reshape(-1).astype(F32))).astype(F32)
    bb = (kf * (F32(ppy) - py.reshape(-1).astype(F32))).astype(F32)
    tiny = F32(F32(1e-30) * kf * kf)
    k0s = F32(k0 - F32(SHIFT))
    Rs = score_fp64.rodrigues(np.asarray(poses6)[:, :3])
    one, zero = np.ones(N, F32), np.zeros(N, F32)
    out = []
    for h, e in enumerate(np.asarray(assign)):
        c = plane_centre(planes[e])
        X = (planes[e] - c[:, None]).astype(F32)
        Xb = tf32_rna(X)
        Xs = tf32_rna(X - Xb)
        R, t = Rs[h], np.asarray(poses6[h, 3:], F64)
        comp = []
        for r in range(3):
            sc = F64(f) * F64(kf) if r < 2 else 1.0
            a = (sc * R[r]).astype(F32)
            b = F32(sc * (R[r] @ c.astype(F64) + t[r]))
            if transform == "fp32":
                comp.append(fma(a[0], X[0], fma(a[1], X[1], fma(a[2], X[2], b))))
                continue
            ab, bb_ = tf32_rna(a), tf32_rna(b)
            as_, bs = tf32_rna(a - ab), tf32_rna(b - bb_)
            d1 = mma([ab[i] * Xb[i] for i in range(3)] + [bb_ * one] + [ab[i] * Xs[i] for i in range(3)] + [bs * one],
                     zero, trunc)
            t2 = [as_[i] * Xb[i] for i in range(3)]
            if transform == "4xtf32":
                t2 += [as_[i] * Xs[i] for i in range(3)]
            comp.append(mma(t2, d1, trunc))
        xc, yc, zc = comp
        pu, pv = fma(aa, zc, xc), fma(bb, zc, yc)
        num = fma(pu, pu, fma(pv, pv, tiny))
        m = ((zc * zc).astype(F32) * num).astype(F32)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            rs = (1.0 / np.sqrt(F64(m))).astype(F32)
            if fold:
                tmax = fma(F32(max_reproj), k1, k0s)
                tt = fma(num, rs, k0s)
                tt = np.where(np.isnan(tt), tmax, np.minimum(tt, tmax))
                d = (np.exp2(F64(tt)).astype(F32) + F32(2.0 ** -SHIFT)).astype(F32)
                da, db = d[0::2], d[1::2]
                pair = ((da + db).astype(F32) * (1.0 / F64((da * db).astype(F32))).astype(F32)).astype(F32)
                w = np.repeat(F64(pair) * 2.0 ** -SHIFT / 2, 2)
            else:
                err = (num * rs).astype(F32)
                err = np.where(np.isnan(err), F32(max_reproj), np.minimum(err, F32(max_reproj)))
                tt = fma(err, k1, k0)
                w = (1.0 / (1.0 + np.exp2(F64(tt)).astype(F32)).astype(F32)).astype(F32)
        out.append(F64(w))
    return np.array(out)


def pair_err(w, ref):
    return np.abs((w[:, 0::2] + w[:, 1::2]) - (ref[:, 0::2] + ref[:, 1::2])).max()


VARIANTS = [("fp32", False, False), ("fp32", False, True)] + [
    (tr, tc, fo) for tr in ("3xtf32", "4xtf32") for fo in (False, True) for tc in (False, True)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", default="480x640,120x160,60x80")
    args = ap.parse_args()
    cases = []
    for name in args.maps.split(","):
        H, W, sub, sx, sy, _ = PROBE_SHAPES[name]
        coords, assign, poses, params = probe_scene(H, W, sub, sx, sy, seed=H + W + sub)
        ref = score_fp64.score(coords, assign, poses, *params)[1].reshape(len(assign), -1)
        cases.append((f"probes {name}", coords, assign, poses, params, ref))
    for name, kw in DENSE.items():
        if kw["H"] * kw["W"] % 2:
            continue
        sc = make_scene(**kw)
        poses = _dense_poses(sc, np.random.default_rng(kw["seed"]), len(sc.assign))
        ref = score_fp64.score(sc.coords, sc.assign, poses, *sc.params)[1].reshape(len(sc.assign), -1)
        cases.append((f"dense {name}", sc.coords, sc.assign, poses, sc.params, ref))
    print("transform  accumulate  fold  | " + " | ".join(c[0] for c in cases))
    for tr, tc, fo in VARIANTS:
        cols = []
        for label, coords, assign, poses, params, ref in cases:
            w = weights(coords, assign, poses, *params, transform=tr, trunc=tc, fold=fo)
            if label.startswith("probes"):
                cols.append(f"{pair_err(w, ref):.2e}")
            else:
                alpha, N = params[6], ref.shape[1]
                cols.append(f"{np.abs(alpha / N * (w.sum(1) - ref.sum(1))).max():.2e}")
        acc = "-" if tr == "fp32" else ("trunc" if tc else "nearest")
        print(f"{tr:9s}  {acc:10s}  {'on' if fo else 'off':4s}  | " + " | ".join(cols), flush=True)


if __name__ == "__main__":
    main()
