"""Writes tests/golden/ref_*.npz: outputs of the reference's OWN compiled code (oracle/_ref/esac_ref = the unmodified
code/esac sources on the real OpenCV of the cv2 wheel, see oracle/build_ref.py), run single-threaded on its
default std::mt19937 stream (seed 1305).

Each fixture holds the scene (small cases) or the make_scene() arguments that regenerate it (480x640 cases: the tensors
are 7-25 MB), every minimal set the reference tried in order (`cells` [M,T,4,2], padded with the accepted set; `tries`), and
the reference's results: winning expert, camera pose, expected loss and the gradient tensor (small cases) or a fixed random
sample of its entries plus per-plane sums (480x640 cases).  tests/test_gpu_ref_golden.py injects the same minimal sets into
the CUDA path and compares; tests/test_oracle.py checks the oracle against them on the CPU.

Needs a checkout of vislearn/esac named by $ESAC_REFERENCE.  Run:  python tests/golden/make_ref_golden.py [name ...]
"""
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from esac_b200.synth import make_scene  # noqa: E402
from oracle import esac_oracle as O  # noqa: E402
from oracle.build_ref import load_ref  # noqa: E402

# pi - 1e-4 about (1, 2, 3)/sqrt(14), as plain floats so that the fixture's scene_kw stays a Python literal
NEAR_PI_RVEC = tuple(float(v) for v in np.array([1.0, 2.0, 3.0]) / np.sqrt(14.0) * (np.pi - 1e-4))
T_MAX = 8  # candidate sets kept per hypothesis (hypotheses that needed more tries keep their LAST T_MAX)
N_SAMPLE = 40000

SMALL = {
    "ref_c1_single_expert_60x80": dict(E=1, H=60, W=80, M=64, sub=8, seed=41),                  # BASELINE configs[0]
    "ref_ensemble3_30x40_shift": dict(E=3, H=30, W=40, M=48, sub=8, seed=42, shiftX=2, shiftY=-3),
    "ref_portrait_40x27": dict(E=2, H=40, W=27, M=32, sub=8, seed=43),
    "ref_world_scale_24x32": dict(E=2, H=24, W=32, M=32, sub=8, seed=48, outdoor=True, world_offset=700.0),
    # the two "clamping for stability" sites (esac.cpp:436-437 max|J_R| > 10, esac_derivative.h:287 max|dPNP| > 10):
    # tiny maps make the minimal sets clustered (dPNP of 9 of 12 hypotheses exceeds 10), lengths in units of 1/7000 m
    # push J_R = -(J^T J)^-1 J^T over 10 for every contributing hypothesis, 1/5000 m keeps it just below
    "ref_clamp_dpnp_9x12": dict(E=1, H=9, W=12, M=12, sub=8, seed=71, outlier_frac=0.1, noise=0.01, alpha=5.0),
    "ref_clamp_jr_on_12x16": dict(E=2, H=12, W=16, M=12, sub=8, seed=63, outlier_frac=0.3, noise=0.002, unit_scale=7000.0),
    "ref_clamp_jr_off_12x16": dict(E=2, H=12, W=16, M=12, sub=8, seed=63, outlier_frac=0.3, noise=0.002, unit_scale=5000.0),
    # cameras far from the world axes (make_scene's own rotations stay within 30 degrees): the half turn about x (y down,
    # looking along world -z) and 1e-4 rad short of a half turn about (1, 2, 3)/sqrt(14), where good hypotheses' rvecs
    # sit at the sign flip of Rodrigues' vector
    "ref_flip_x_30x40": dict(E=2, H=30, W=40, M=32, sub=8, seed=1, rotation=(3.141592653589793, 0.0, 0.0)),
    "ref_near_pi_30x40": dict(E=2, H=30, W=40, M=32, sub=8, seed=1, rotation=NEAR_PI_RVEC),
}
LARGE = {
    "ref_mid_4x120x160": dict(E=4, H=120, W=160, M=48, sub=4, seed=45),
    "ref_full_7x480x640": dict(E=7, H=480, W=640, M=32, sub=1, seed=46, active_only=False),       # BASELINE configs[1] shape
    "ref_full_world_2x480x640": dict(E=2, H=480, W=640, M=16, sub=1, seed=47, outdoor=True, world_offset=700.0),
}
LOSS_ARGS = (1.0, 100.0, 100.0)  # wLossRot, wLossTrans, lossCut (train_esac.py:44-50 defaults)


def tried_sets(sc, seed=1305):
    """Replays the reference's sampling on the oracle (identical stream, identical verdicts -- tests/test_ref_pin.py) and
    records every candidate set."""
    log = []
    orig = O.draw_minimal_set_mt

    def rec(mt, W, H):
        c = orig(mt, W, H)
        log.append(c)
        return c

    O.draw_minimal_set_mt = rec
    try:
        K = O.cam_mat(sc.f, sc.ppx, sc.ppy)
        E, _, H, W = sc.coords.shape
        hyps = O.sample_hypotheses(sc.coords, sc.assign, O.create_sampling(W, H, sc.sub, sc.shiftX, sc.shiftY), K,
                                   O.MAX_SAMPLING_TRIES, sc.tau, mt=O.ThreadRandStream(seed))
    finally:
        O.draw_minimal_set_mt = orig
    tries = np.array([h.tries for h in hyps], np.int32)
    M = len(hyps)
    cells = np.zeros((M, T_MAX, 4, 2), np.int32)
    pos = 0
    for h in range(M):
        mine = log[pos:pos + tries[h]]
        pos += tries[h]
        mine = mine[-T_MAX:]
        for t in range(T_MAX):
            cells[h, t] = np.array(mine[min(t, len(mine) - 1)], np.int32)
    assert pos == len(log)
    return cells, tries


def run_reference(R, sc):
    co, asg = torch.from_numpy(sc.coords), torch.from_numpy(sc.assign)
    R.force_init(1305)
    pose = torch.zeros(4, 4)
    t0 = time.time()
    e = R.forward(co, asg, pose, *sc.params)
    t1 = time.time()
    R.force_init(1305)
    g = torch.zeros(sc.coords.shape)
    loss = R.backward(co, g, asg, torch.from_numpy(sc.gt_pose), *LOSS_ARGS, *sc.params)
    t2 = time.time()
    return e, pose.numpy(), loss, g.numpy(), (t1 - t0, t2 - t1)


if __name__ == "__main__":
    here = Path(__file__).resolve().parent
    R = load_ref()
    assert R is not None, "needs $ESAC_REFERENCE"
    R.set_num_threads(1)
    R.set_native_project(False)
    want = set(sys.argv[1:])
    for name, kw in {**SMALL, **LARGE}.items():
        if want and name not in want:
            continue
        sc = make_scene(**kw)
        cells, tries = tried_sets(sc)
        e, pose, loss, g, dt = run_reference(R, sc)
        # auxiliary: the oracle's per-hypothesis view of the same run (the reference does not expose scores); the
        # generator refuses to write a fixture on which oracle and reference disagree
        o_pose = np.zeros((4, 4), np.float32)
        o_e, tr = O.forward(sc.coords, sc.assign, o_pose, *sc.params, mt=O.ThreadRandStream(1305), trace=True)
        assert o_e == e and np.abs(o_pose - pose).max() <= 1e-6, (name, o_e, e, np.abs(o_pose - pose).max())
        top = np.sort(np.array(tr.scores))[::-1]
        assert top[0] - top[1] > 1e-2, f"{name}: near-tie at the top ({top[0] - top[1]:.2e}) -- pick another seed"
        # which hypotheses trip the two clamps, and how far the gradient would move without them (oracle view)
        g_o = np.zeros_like(sc.coords)
        _, bt = O.backward(sc.coords, g_o, sc.assign, sc.gt_pose, *LOSS_ARGS, *sc.params, mt=O.ThreadRandStream(1305), trace=True)
        extra = {}
        if name.startswith("ref_clamp"):
            g_u = np.zeros_like(sc.coords)
            O.backward(sc.coords, g_u, sc.assign, sc.gt_pose, *LOSS_ARGS, *sc.params, mt=O.ThreadRandStream(1305),
                       clamp_thresh=np.inf)
            extra = dict(clamped_jr=np.array(bt.clamped_jr, np.int32), clamped_dpnp=np.array(bt.clamped_dpnp, np.int32),
                         unclamped_grad_diff=float(np.abs(g_u - g_o).max()))
            print(f"  clamps: J_R {bt.clamped_jr}, dPNP {bt.clamped_dpnp}, |g(no clamp) - g| max {extra['unclamped_grad_diff']:.3g}")
        common = dict(**extra, scene_kw=np.array(repr(kw)), assign=sc.assign, gt_pose=sc.gt_pose, params=np.array(sc.params, np.float64),
                      loss_args=np.array(LOSS_ARGS), cells=cells, tries=tries, expert=e, pose=pose, loss=loss,
                      oracle_scores=np.array(tr.scores), oracle_winner=tr.winner, oracle_rounds=tr.rounds,
                      oracle_inliers=int(tr.inlier_map.sum()) if tr.inlier_map is not None else 0)
        if name in SMALL:
            np.savez_compressed(here / f"{name}.npz", coords=sc.coords, grads=g, **common)
        else:
            rng = np.random.default_rng(7)
            nz = np.flatnonzero(g.reshape(-1))
            idx = np.sort(np.concatenate([rng.choice(g.size, N_SAMPLE // 2, replace=False),
                                          rng.choice(nz, min(N_SAMPLE // 2, nz.size), replace=False)])).astype(np.int64)
            np.savez_compressed(here / f"{name}.npz", grad_idx=idx, grad_val=g.reshape(-1)[idx],
                                grad_plane_sum=g.astype(np.float64).sum(axis=(2, 3)), grad_plane_abs=np.abs(g).astype(np.float64).sum(axis=(2, 3)),
                                grad_max=np.abs(g).max(), coords_sum=sc.coords.astype(np.float64).sum(), **common)
        print(f"{name}: expert {e} loss {loss:.9f} |g|max {np.abs(g).max():.4g} tries max {tries.max()} "
              f"(reference fwd {dt[0]:.1f}s bwd {dt[1]:.1f}s)", flush=True)
