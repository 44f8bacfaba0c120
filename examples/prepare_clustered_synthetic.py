"""From an SfM reconstruction to a clustered environment: a synthetic Aachen-like reconstruction
(esac_b200.synth.make_reconstruction) is rendered on the device and written as a training set (init / poses /
calibration, esac_b200.prepare.write_training_set, in place of setup_aachen.py's render loop), then the rendered maps are
clustered into experts (esac_b200.cluster.cluster_environment, in place of cluster_dataset.py).

    python examples/prepare_clustered_synthetic.py --cameras 500 --points 150000 --clusters 10 --check

--check renders the same reconstruction with the numpy restatement in oracle/render_oracle.py (render_fixed), compares
every map bitwise with the files written, and clusters its maps too: the labels must agree exactly.
"""
from __future__ import annotations

import argparse
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from esac_b200 import prepare  # noqa: E402
from esac_b200.cluster import cluster_environment  # noqa: E402
from esac_b200.synth import make_reconstruction  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, default=500)
    ap.add_argument("--points", type=int, default=150_000)
    ap.add_argument("--clusters", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args(argv)
    r = make_reconstruction(a.seed, a.cameras, a.points)
    rec = r["rec"]
    with tempfile.TemporaryDirectory() as dst:
        t = time.perf_counter()
        out = prepare.write_training_set(dst, rec, r["sizes"])
        t_write = time.perf_counter() - t
        clustering = cluster_environment(out.maps, a.clusters, seed=a.seed)
        sizes = torch.bincount(clustering.labels, minlength=a.clusters).tolist()
        print(f"{len(out.names)} cameras, {int(rec.offsets[-1])} observations rendered and written in {t_write:.2f} s; "
              f"{int(out.counts.sum())} cells hold a point; cluster sizes {sizes}")
        if a.check:
            from oracle.render_oracle import render_fixed
            want = render_fixed(rec.points, rec.offsets, rec.indices, rec.poses, rec.focal, r["out_scale"], r["shapes"])[0]
            for name, m in zip(out.names, want):
                saved = torch.load(Path(dst) / "init" / (name[:-4] + ".dat"))
                if not np.array_equal(saved.numpy().view(np.uint32), m.view(np.uint32)):
                    raise SystemExit(f"check failed: {name} differs from render_fixed")
            other = cluster_environment([torch.from_numpy(m) for m in want], a.clusters, seed=a.seed)
            if not torch.equal(other.labels.cpu(), clustering.labels.cpu()):
                raise SystemExit("check failed: the clustering of render_fixed's maps differs")
            print(f"check: {len(want)} maps bitwise equal to render_fixed, identical cluster labels")


if __name__ == "__main__":
    main()
