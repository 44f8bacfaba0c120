"""Writes tests/golden/pin/ref_pose_loss_edges.npz: what the reference's OWN loss() and dLoss() (esac_loss.h, compiled into
oracle/_ref/esac_ref, see oracle/build_ref.py) return on the pose-loss edge grid of tests/pose_loss_grid.py.

Per ground-truth orientation `<name>`:
  <name>_poses   float64 [N, 6]  the estimates (rvec, tvec)
  <name>_cuts    float64 [N]     the cut of each entry (float32 values; "equal" entries hold the loss at cut off)
  <name>_loss    float64 [N]     loss(pose2trans(estimate), ground truth)
  <name>_dloss   float64 [N, 6]  dLoss(estimate, trans2pose(ground truth))
  <name>_class   int32 [N, 6]    union of the outcome classes (1 zero, 2 finite, 4 non-finite) of dLoss over the estimate
                                 and its nudged copies (pose_loss_grid.nudged), i.e. every class rounding can lead the
                                 reference to at that entry
The ground truths are pose_loss_grid.ground_truth(name); the loss weights are pose_loss_grid.W_ROT / W_TRANS.

Needs a checkout of vislearn/esac named by $ESAC_REFERENCE.  Run:  python tests/golden/make_ref_pose_loss_pin.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from oracle import esac_oracle as O  # noqa: E402
from oracle.build_ref import load_ref  # noqa: E402
from orientations import NAMES  # noqa: E402
from pose_loss_grid import CUT_OFF, W_ROT, W_TRANS, classes, cut_value, estimates, ground_truth, nudged  # noqa: E402

OUT = Path(__file__).resolve().parent / "pin" / "ref_pose_loss_edges.npz"


def pin_orientation(R, name):
    gt = ground_truth(name)
    T2 = gt.astype(np.float64).ravel().tolist()
    r2, t2 = O.trans2pose(gt)
    gt6 = np.concatenate([r2.ravel(), t2.ravel()]).tolist()
    poses, keys = estimates(gt)
    cuts, losses, dl, cls = [], [], [], []
    for est, key in zip(poses, keys):
        T1 = O.pose2trans(est[:3], est[3:]).ravel().tolist()
        cut = cut_value(key, R.loss(T1, T2, W_ROT, W_TRANS, CUT_OFF))
        cuts.append(cut)
        losses.append(R.loss(T1, T2, W_ROT, W_TRANS, cut))
        d = np.array(R.d_loss(est.tolist(), gt6, W_ROT, W_TRANS, cut))
        dl.append(d)
        c = classes(d)
        for e in nudged(est):
            c = c | classes(R.d_loss(e.tolist(), gt6, W_ROT, W_TRANS, cut))
        cls.append(c)
    return {f"{name}_poses": poses, f"{name}_cuts": np.array(cuts), f"{name}_loss": np.array(losses),
            f"{name}_dloss": np.array(dl), f"{name}_class": np.array(cls, np.int32)}


if __name__ == "__main__":
    R = load_ref()
    assert R is not None, "needs $ESAC_REFERENCE"
    out = {}
    for name in NAMES:
        out.update(pin_orientation(R, name))
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), "arrays")
