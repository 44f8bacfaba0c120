"""test_esac.py on the device in one command (python -m esac_b200.localize): on synthetic environments written under
tmp_path -- a room environment of three scenes with images of two shapes, and a clustered environment -- the results and
pose files equal those of an eager loop of the same library calls (the image set's step, GatingNet, assign_hypotheses with
the same seeds, ExpertStack.forward, esac.forward, PoseEvaluator), with and without -es, with -os, and with -c."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import localize
from esac_b200.data import ClusterDraws, RoomDraws, cluster_jitter, from_cluster_folder, from_room_folders
from esac_b200.evaluate import PoseEvaluator
from esac_b200.experts import ExpertStack
from esac_b200.gating_net import GatingNet
from oracle import expert_oracle as XO
from oracle import gating_oracle as GO

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


def write_environment(root: Path, scenes: int, shapes, seed: int):
    """Scene folders with test/{rgb,poses,calibration} files, and env_list.txt naming them."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    names = []
    for s in range(scenes):
        base = root / f"scene{s}" / "test"
        for sub in ("rgb", "poses", "calibration"):
            (base / sub).mkdir(parents=True)
        for j, (h, w) in enumerate(shapes):
            low = rng.random((h // 8, w // 8, 3))
            img = np.kron(low, np.ones((8, 8, 1))) * 200 + rng.random((h, w, 3)) * 40
            Image.fromarray(img.clip(0, 255).astype(np.uint8)).save(base / "rgb" / f"frame-{j:06d}.color.png")
            pose = np.eye(4)
            pose[:3, 3] = rng.normal(size=3)
            np.savetxt(base / "poses" / f"frame-{j:06d}.pose.txt", pose)
            np.savetxt(base / "calibration" / f"frame-{j:06d}.calibration.txt", [525.0 + 10 * j])
        names.append(str(root / f"scene{s}"))
    (root / "env_list.txt").write_text("".join(n + "\n" for n in names))


def write_ensemble(path: Path, E: int, capacity: int, seed: int):
    """An ensemble file as ExpertEnsemble.save writes it: [gating state dict, expert state dicts...]."""
    sds = [GO.kaiming_state_dict(seed, E, capacity)]
    sds += [XO.kaiming_state_dict(seed + 1 + e, mean=(0.3 * e, -0.5, 2.0 + 0.2 * e)) for e in range(E)]
    torch.save(sds, path)
    return sds


def run_localize(cwd: Path, *args):
    env = dict(os.environ, PYTHONPATH=str(ROOT) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "esac_b200.localize", *args], cwd=cwd, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def eager_files(cwd: Path, sds, clustered: bool, es=False, os_=False, seed=0, M=256):
    """The results and pose lines of the eager loop of the same library calls."""
    prev = Path.cwd()
    os.chdir(cwd)
    try:
        ds = from_cluster_folder("test", training=False) if clustered else from_room_folders("test", training=False)
        files = localize.rgb_files(clustered)
    finally:
        os.chdir(prev)
    E = len(sds) - 1
    gating, stack = GatingNet(sds[0], "cuda"), ExpertStack(sds[1:], "cuda")
    draws = ClusterDraws(len(ds), jitter=cluster_jitter(False)) if clustered else RoomDraws(ds.scene_counts, training=False)
    plan = ds.plan(draws, batch=1, shuffle=False, shift=False)
    ds.load_plan(plan)
    ev = PoseEvaluator(E, len(ds), clustered=clustered)
    api.context().set_option("fixed_seed", 0)
    api.set_seed(seed)
    for i, g in enumerate(plan.groups):
        out = ds.step(g)
        log_p, probs = torch.empty(1, E, device="cuda"), torch.empty(1, E, device="cuda")
        gating.forward_async(out["image"], log_p, probs)
        if os_:
            probs = torch.nn.functional.one_hot(out["scenes"], E).float()
        e_hyps, hist = api.assign_hypotheses(probs, M, seed + i, expertSelection=es or os_)
        pred = stack.forward(out["image"], hist)
        pose = torch.zeros(4, 4, device="cuda")
        (sx, sy), (f, ppx, ppy) = out["shifts"][0].tolist(), out["cameras"][0].tolist()
        e = api.forward(pred[0], e_hyps[0], pose, sx, sy, f, ppx, ppy, 10.0, 100.0, 0.5, 100.0, 8)
        ev.update(pose[None], out["gt_poses"], torch.tensor([e], device="cuda"), out["scenes"], hist=hist,
                  status=torch.zeros(1, dtype=torch.int32, device="cuda"))
    t = ev.table(5, 5, average=not clustered)
    return t["results"], ev.pose_lines([localize.strip_file_name(f) for f in files])


def read_lines(path: Path):
    return path.read_text().splitlines()


def test_room_environment(tmp_path):
    write_environment(tmp_path, 3, [(48, 64), (64, 48)], seed=1)
    sds = write_ensemble(tmp_path / "esac_syn.net", 3, 1, seed=10)
    write_ensemble(tmp_path / "es_syn.net", 3, 1, seed=20)
    out = run_localize(tmp_path, "-sid", "syn", "--seed", "7")
    assert "Environment has 6 test images." in out and "Avg. Time:" in out and "Average" in out
    results, poses = eager_files(tmp_path, sds, False, seed=7)
    assert read_lines(tmp_path / "results_esac_syn.txt") == results
    assert read_lines(tmp_path / "poses_esac_syn.txt") == poses
    assert len(poses) == 6 and poses[0].startswith("frame-000000.color.png ")

    run_localize(tmp_path, "-sid", "syn", "-es", "--seed", "3")
    results, poses = eager_files(tmp_path, torch.load(tmp_path / "es_syn.net"), False, es=True, seed=3)
    assert read_lines(tmp_path / "results_esac_es_syn.txt") == results
    assert read_lines(tmp_path / "poses_esac_es_syn.txt") == poses

    run_localize(tmp_path, "-sid", "syn", "-os")
    results, poses = eager_files(tmp_path, sds, False, os_=True)
    assert read_lines(tmp_path / "results_esac_os_syn.txt") == results
    assert read_lines(tmp_path / "poses_esac_os_syn.txt") == poses
    # oracle selection: every image's hypotheses go to its own scene's expert
    assert all(float(line.split()[0]) == 1.0 for line in results)


def test_clustered_environment(tmp_path):
    write_environment(tmp_path, 1, [(48, 64), (48, 64), (64, 48), (48, 64)], seed=2)
    sds = write_ensemble(tmp_path / "esac_cl.net", 2, 2, seed=30)
    out = run_localize(tmp_path, "-c", "2", "-sid", "cl", "-hyps", "128")
    assert "Environment has 4 test images." in out and "Average" not in out
    results, poses = eager_files(tmp_path, sds, True, M=128)
    assert read_lines(tmp_path / "results_esac_cl.txt") == results
    assert read_lines(tmp_path / "poses_esac_cl.txt") == poses
    r = subprocess.run([sys.executable, "-m", "esac_b200.localize", "-c", "2", "-os"], cwd=tmp_path, capture_output=True,
                       text=True, env=dict(os.environ, PYTHONPATH=str(ROOT)))
    assert r.returncode != 0 and "clustered environment" in r.stderr
