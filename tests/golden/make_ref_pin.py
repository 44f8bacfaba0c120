"""Writes tests/golden/pin/ref_pin.npz: what the reference's OWN compiled code (oracle/_ref/esac_ref, see
oracle/build_ref.py) returns for the calls of tests/test_ref_pin.py, single-threaded on its default std::mt19937 stream.
The file has a directory of its own so that the fixture globs over tests/golden/*.npz do not pick it up.

Needs a checkout of vislearn/esac named by $ESAC_REFERENCE.  Run:  python tests/golden/make_ref_pin.py
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from esac_b200.synth import make_scene  # noqa: E402
from oracle.build_ref import load_ref  # noqa: E402
from test_ref_pin import CASES, CUT_CASES, CUT_SCENE, IRAND_MAX, PERSIST_SCENE  # noqa: E402

if __name__ == "__main__":
    R = load_ref()
    assert R is not None, "needs $ESAC_REFERENCE"
    R.set_num_threads(1)
    R.set_native_project(False)
    out = {}
    R.force_init(1305)
    out["irand_1305"] = np.array([[R.irand(0, m, 0) for _ in range(300)] for m in IRAND_MAX], np.int64)
    R.force_init(77)
    out["irand_77"] = np.array([R.irand(3, 11, 0) for _ in range(50)], np.int64)
    for name, kw in CASES.items():
        sc = make_scene(**kw)
        co, asg = torch.from_numpy(sc.coords), torch.from_numpy(sc.assign)
        R.force_init(1305)
        pose = torch.zeros(4, 4)
        out[f"{name}_expert"] = R.forward(co, asg, pose, *sc.params)
        out[f"{name}_pose"] = pose.numpy()
        R.force_init(1305)
        g = torch.full(sc.coords.shape, 0.25)
        out[f"{name}_loss"] = R.backward(co, g, asg, torch.from_numpy(sc.gt_pose), 1.0, 100.0, 100.0, *sc.params)
        out[f"{name}_grads"] = g.numpy()
    sc = make_scene(**CUT_SCENE)
    gt = sc.gt_pose.copy()
    gt[:3, 3] += np.array([3.0, -2.0, 1.0], np.float32)
    for i, (w_rot, w_trans, cut) in enumerate(CUT_CASES):
        R.force_init(1305)
        g = torch.zeros(sc.coords.shape)
        out[f"cut{i}_loss"] = R.backward(torch.from_numpy(sc.coords), g, torch.from_numpy(sc.assign), torch.from_numpy(gt),
                                         w_rot, w_trans, cut, *sc.params)
        out[f"cut{i}_grads"] = g.numpy()
    sc = make_scene(**PERSIST_SCENE)
    R.force_init(1305)
    poses = []
    for _ in range(2):
        pose = torch.zeros(4, 4)
        R.forward(torch.from_numpy(sc.coords), torch.from_numpy(sc.assign), pose, *sc.params)
        poses.append(pose.numpy())
    out["persist_poses"] = np.stack(poses)
    np.savez_compressed(Path(__file__).resolve().parent / "pin" / "ref_pin.npz", **out)
    print(sorted(out))
