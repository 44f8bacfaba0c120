"""How good a cut the prefilter's "near-certain" hint makes (option sample_hint), on the host compile.  CPU only.

prefilter_kernel stops prefiltering a hypothesis' window after a surviving try the float path puts within sample_hint * tau
on the 4th point (esac_b200/csrc/hyp.cu).  What that saves depends on two rates, measured here on bench-shaped tries (the
bench's scenes: 7 experts, 480x640 maps, subSampling 1, tau 10; tries are 4 distinct random cells of one expert's map):

  precision  P(accept | hint): a hinted try the exact verdict rejects costs a resume (the window restarts after it)
  coverage   P(hint | accept): an accepted try without a hint cuts nothing

per expert kind (the true expert, where most tries pass, and the wrong ones, where ~1e-3 do).

  python tools/sample_cut_ab.py [--tries N] [--hints 0.5 0.75 0.9]
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from esac_b200.api import load_library  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402


def draws(sc, e, n, rng):
    _, _, H, W = sc.coords.shape
    xs = rng.integers(0, W - 1, (n, 4))
    ys = rng.integers(0, H - 1, (n, 4))
    key = np.sort(ys * W + xs, axis=1)
    ok = (np.diff(key, axis=1) != 0).all(axis=1)
    xs, ys = xs[ok], ys[ok]
    obj = np.ascontiguousarray(sc.coords[e][:, ys, xs].transpose(1, 2, 0), np.float32)
    img = np.ascontiguousarray(np.stack([xs * sc.sub + sc.sub // 2 - sc.shiftX, ys * sc.sub + sc.sub // 2 - sc.shiftY], -1),
                               np.float32)
    return obj, img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tries", type=int, default=200000, help="tries per expert kind")
    ap.add_argument("--hints", type=float, nargs="+", default=[0.5, 0.75, 0.9])
    ap.add_argument("--seed", type=int, default=100)
    args = ap.parse_args()
    lib = load_library()
    sc = make_scene(E=7, H=480, W=640, M=256, sub=1, seed=args.seed, per_expert=True, active_only=False)
    rng = np.random.default_rng(args.seed)
    kinds = {"true": [sc.gt_expert], "wrong": [e for e in range(7) if e != sc.gt_expert]}
    print(f"bench scene seed {args.seed}: tau {sc.tau}, f {sc.f}, {args.tries} tries per kind")
    print(f"{'kind':6} {'hint':>5} {'tries':>8} {'survive':>8} {'accept':>7} {'hinted':>7} {'prec':>7} {'cover':>7}")
    for kind, experts in kinds.items():
        per = args.tries // len(experts)
        sets = [draws(sc, e, per, rng) for e in experts]
        obj = np.concatenate([s[0] for s in sets])
        img = np.concatenate([s[1] for s in sets])
        n = len(obj)
        for h in args.hints:
            mp, hi, ac = (np.zeros(n, np.int32) for _ in range(3))
            lib.esacb200_host_tries_hint(n, obj.ctypes.data, img.ctypes.data, sc.f, sc.ppx, sc.ppy, sc.tau, h, mp.ctypes.data,
                                         hi.ctypes.data, ac.ctypes.data)
            mp, hi, ac = mp.astype(bool), hi.astype(bool), ac.astype(bool)
            assert not (hi & ~mp).any() and not (ac & ~mp).any()
            prec = (hi & ac).sum() / max(hi.sum(), 1)
            cover = (hi & ac).sum() / max(ac.sum(), 1)
            print(f"{kind:6} {h:5.2f} {n:8d} {mp.sum():8d} {ac.sum():7d} {hi.sum():7d} {prec:7.3f} {cover:7.3f}")


if __name__ == "__main__":
    main()
