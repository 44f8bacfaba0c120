"""test_esac.py's evaluation (code/test_esac.py:209-289) on the device, in a record store a captured test step writes to.

    ev = PoseEvaluator(num_scenes=E, capacity=len(testset))
    # inside the captured step, after api.forward_async(..., pose, expert, status):
    ev.update(pose, gt_pose, expert, gt_scene, hist=hist, status=status)
    # after the loop, the one read-back:
    t = ev.table()
    print("\\n".join(t["console"]))

update() enqueues one kernel on torch's current stream (api.evaluate_poses_async) that writes each image's record (pose
errors, correct expert, experts active, pose-file entry; api.EVAL_FIELDS) to the next free row; the row counter lives on
the device, so every replay of a captured update appends.  records() reads the store back once; table() and pose_lines()
format it as the reference prints and writes it.

An image whose forward status is not 0, or whose scene lies outside [0, num_scenes), keeps its record but is left out of
the table and counted in table()["excluded"]: the reference cannot produce such images.  The experts-active figures average
over the counted images.

A clustered environment (test_esac.py with --clusters, a SyntheticClusterDataset or a clustering of esac_b200.cluster) has
no ground-truth expert: its images carry scene -1.  PoseEvaluator(..., clustered=True) counts every record with status 0
in scene 0, whatever its scene, as test_esac.py's cluster mode does: one row, whose class accuracy is 0 since -1 matches
no expert.  Read it with table(average=False), the cluster mode's console.
"""
from __future__ import annotations

import numpy as np

from . import api

_ROT, _TRANS, _CORRECT, _SCENE, _STATUS, _ACTIVE = 0, 1, 2, 3, 5, 6
_RULE = "-" * 60


class PoseEvaluator:
    """Records of up to `capacity` test images of `num_scenes` scenes (the ensemble's experts), on `device` (default: the
    current CUDA device)."""

    def __init__(self, num_scenes: int, capacity: int, device=None, clustered: bool = False):
        import torch
        if int(num_scenes) < 1 or int(capacity) < 1:
            raise RuntimeError(f"PoseEvaluator needs num_scenes >= 1 and capacity >= 1, got {num_scenes} and {capacity}")
        self.num_scenes = int(num_scenes)
        self.capacity = int(capacity)
        self.clustered = bool(clustered)
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.state = torch.zeros(api.EVAL_STATE, dtype=torch.int64, device=device)
        self.buffer = torch.empty((self.capacity, len(api.EVAL_FIELDS)), dtype=torch.float64, device=device)

    def update(self, outPoses, gtPoses, experts, gtScenes, hist=None, status=None):
        """Appends the records of a batch (api.evaluate_poses_async's arguments) on torch's current stream; capturable."""
        api.evaluate_poses_async(outPoses, gtPoses, experts, gtScenes, self.buffer, self.state, hist=hist, status=status)

    def reset(self):
        """Empties the store, ordered on torch's current stream."""
        self.state.zero_()

    def records(self) -> np.ndarray:
        """The records written so far, float64 [n, 14] (api.EVAL_FIELDS).  Raises when more images were evaluated than
        the store holds."""
        count, overflow = (int(v) for v in self.state[:2].cpu())
        if overflow:
            raise RuntimeError(f"PoseEvaluator: {count} images evaluated into a store of capacity {self.capacity}; the "
                               f"records past row {self.capacity} were dropped")
        return self.buffer[:count].cpu().numpy()

    def table(self, rot_threshold: float = 5, trans_threshold: float = 5, average: bool = True) -> dict:
        """The reference's statistics over the counted records: "rows" (scene, class accuracy, pose accuracy, median
        rotation error in degrees, median translation error in cm), "console" (the lines test_esac.py prints, with the
        Average row when `average`, as for clusters < 0), "results" (the results-file lines), "experts" (the experts-active
        lines) and "excluded" (records left out).  When clustered: one row, scene 0, over every record with status 0."""
        return _table(self.records(), self.num_scenes, rot_threshold, trans_threshold, average, self.clustered)

    def pose_lines(self, names) -> list[str]:
        """The pose-file lines, one per record, names[i] being record i's already stripped file name."""
        recs = self.records()
        if len(names) != len(recs):
            raise RuntimeError(f"pose_lines: {len(names)} names for {len(recs)} records")
        return ["%s %f %f %f %f %f %f %f" % (n, *(float(v) for v in r[7:14])) for n, r in zip(names, recs)]


def _upper_median(values: np.ndarray) -> float:
    """test_esac.py's median: sorted(l)[int(len(l) / 2)], 0 for no value."""
    return float(np.sort(values)[len(values) // 2]) if len(values) else 0


def _table(recs: np.ndarray, num_scenes: int, rot_threshold, trans_threshold, average: bool, clustered: bool = False) -> dict:
    scene = recs[:, _SCENE]
    if clustered:
        counted = recs[:, _STATUS] == 0
        scene = np.where(counted, 0.0, scene)
        num_scenes = 1
    else:
        counted = (recs[:, _STATUS] == 0) & (scene >= 0) & (scene < num_scenes)
    rows, console, results = [], ["Scene - Class.Acc. - Pose.Acc. - Median Rot. - Median Trans.", _RULE], []
    for s in range(num_scenes):
        r = recs[counted & (scene == s)]
        n = max(len(r), 1)
        class_acc = int((r[:, _CORRECT] == 1).sum()) / n
        pose_acc = int(((r[:, _TRANS] < trans_threshold) & (r[:, _ROT] < rot_threshold)).sum()) / n
        row = (s, class_acc, pose_acc, _upper_median(r[:, _ROT]), _upper_median(r[:, _TRANS]))
        rows.append(row)
        console.append("%7d %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (s, class_acc * 100, pose_acc * 100, row[3], row[4]))
        results.append("%f %f %f %f" % row[1:])
    if average:
        sums = [sum(row[i] for row in rows) for i in range(1, 5)]
        console += [_RULE, "Average %7.1f%% %10.1f%% %10.2fdeg %10.2fcm" % (
            sums[0] * 100 / num_scenes, sums[1] * 100 / num_scenes, sums[2] / num_scenes, sums[3] / num_scenes)]
    active = recs[counted, _ACTIVE]
    avg_active = float(active.sum()) / max(len(active), 1)
    max_active = float(active.max()) if len(active) else 0.0
    return {"rows": rows, "console": console, "results": results,
            "experts": [f"Avg. experts active: {avg_active}", f"Max. experts active: {max_active}"],
            "excluded": int((~counted).sum())}
