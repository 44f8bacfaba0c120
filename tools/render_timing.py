"""Times rendering the ground-truth maps of an Aachen-sized reconstruction (about 4 000 cameras with 60x80, 80x60 and
60x107 out maps, 1.5 M points, about 8 M observations; esac_b200.synth.make_reconstruction from a seed), step by step:

* parse: esac_b200.prepare.read_nvm on the reconstruction written as an NVM file;
* render: api.render_init_maps with the points and observations already on the device, CUDA events around each call
  (warm-up first; median, min and max of the repeats), and the whole call from host arrays on the host clock;
* write: prepare.write_training_set (render, then 4 000 init / pose / calibration files) into a temporary directory;
* serial: the reference's per-observation loop (oracle/render_oracle.py render_serial with torch.mm) on the first cameras
  up to a 20 000-observation sample, extrapolated per observation to the whole reconstruction.

Prints one JSON line with the GPU's name and power limit, read in the same run.

    python tools/render_timing.py [--seed 0] [--repeats 10] [--sample 20000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import esac_b200.api as api  # noqa: E402
from esac_b200 import prepare  # noqa: E402
from esac_b200.synth import make_reconstruction  # noqa: E402
from oracle.render_oracle import render_serial  # noqa: E402


def gpu_name_power():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def write_nvm(path, rec):
    """rec as an NVM file (camera: name f qw qx qy qz centre k 0; point: x y z rgb n (camera key x y)*)."""
    from scipy.spatial.transform import Rotation
    C = len(rec.names)
    lines = ["NVM_V3", "", str(C)]
    for c in range(C):
        R = rec.poses[c, :3, :3].astype(np.float64)
        x, y, z, w = (float(t) for t in Rotation.from_matrix(R).as_quat())
        if w < 0:
            w, x, y, z = -w, -x, -y, -z
        centre = [float(t) for t in -R.T @ rec.poses[c, :3, 3].astype(np.float64)]
        lines.append(f"{rec.images[c]} {float(rec.focal[c])!r} {w!r} {x!r} {y!r} {z!r} {centre[0]!r} {centre[1]!r} {centre[2]!r} 0 0")
    P = len(rec.points)
    cams = np.repeat(np.arange(C), np.diff(rec.offsets))
    order = np.argsort(rec.indices, kind="stable")
    per_point = np.split(cams[order], np.cumsum(np.bincount(rec.indices, minlength=P))[:-1])
    lines += ["", str(P)]
    for j in range(P):
        v = per_point[j]
        x, y, z = (float(t) for t in rec.points[j])
        lines.append(f"{x!r} {y!r} {z!r} 0 0 0 {len(v)} "
                     + " ".join(f"{c} 0 0 0" for c in v))
    lines += ["", "0", ""]
    with open(path, "w") as f:
        f.write("\n".join(lines))
    with open(str(path) + ".list.txt", "w") as f:
        f.write("".join(n + "\n" for n in rec.images))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--cameras", type=int, default=4000)
    ap.add_argument("--points", type=int, default=1_500_000)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--sample", type=int, default=20000)
    a = ap.parse_args()
    r = make_reconstruction(a.seed, a.cameras, a.points)
    rec, sizes = r["rec"], r["sizes"]
    V = int(rec.offsets[-1])
    res = {"gpu": gpu_name_power(), "cameras": len(rec.names), "points": len(rec.points), "observations": V}
    with tempfile.TemporaryDirectory() as tmp:
        nvm = os.path.join(tmp, "recon.nvm")
        write_nvm(nvm, rec)
        t = time.perf_counter()
        parsed = prepare.read_nvm(nvm, nvm + ".list.txt")
        res["parse_s"] = time.perf_counter() - t
        assert np.array_equal(parsed.offsets, rec.offsets) and np.array_equal(parsed.indices, rec.indices)

        args = (rec.points, rec.offsets, rec.indices, rec.poses, rec.focal, r["out_scale"], r["shapes"])
        dev_args = (torch.from_numpy(rec.points).cuda(), rec.offsets, torch.from_numpy(rec.indices).cuda()) + args[3:]
        api.render_init_maps(*dev_args)
        ms = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            maps, _, _ = api.render_init_maps(*dev_args)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
            del maps
        res["render_device_inputs_ms"] = {"median": float(np.median(ms)), "min": float(min(ms)), "max": float(max(ms))}
        host = []
        for _ in range(max(3, a.repeats // 3)):
            t = time.perf_counter()
            maps, _, _ = api.render_init_maps(*args)
            torch.cuda.synchronize()
            host.append((time.perf_counter() - t) * 1e3)
            del maps
        res["render_host_inputs_wall_ms"] = {"median": float(np.median(host)), "min": float(min(host)),
                                             "max": float(max(host))}

        t = time.perf_counter()
        out = prepare.write_training_set(os.path.join(tmp, "training"), rec, sizes)
        res["write_training_set_s"] = time.perf_counter() - t
        res["files_written"] = len(out.names)

    n_cam = int(np.searchsorted(rec.offsets, a.sample, "left"))
    n_cam = max(1, n_cam)
    sub = (rec.points, rec.offsets[:n_cam + 1], rec.indices[:int(rec.offsets[n_cam])], rec.poses[:n_cam],
           rec.focal[:n_cam], r["out_scale"][:n_cam], r["shapes"][:n_cam])
    t = time.perf_counter()
    render_serial(*sub, product="torch")
    dt = time.perf_counter() - t
    n_obs = int(rec.offsets[n_cam])
    res["serial_sample_observations"] = n_obs
    res["serial_us_per_observation"] = dt / n_obs * 1e6
    res["serial_extrapolated_s"] = dt / n_obs * V
    print(json.dumps(res))


if __name__ == "__main__":
    main()
