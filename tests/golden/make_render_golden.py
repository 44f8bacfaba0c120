"""Writes tests/golden/render/*.npz: small synthetic SfM reconstructions and what the reference's converters make of them.

The converters are datasets/setup_aachen.py's create_training_set and datasets/setup_dubrovnik.py's create_set, run
unmodified from the reference checkout ($ESAC_REFERENCE, else a checkout named `reference` beside the repository).  Both
scripts download at import time, so each function is taken from the script's AST and executed with its module globals
stubbed: the file names, the folders, `opt`, the image list, `mkdir`, and an `os` whose `system` does nothing (no links).
A proxy `torch` records what the function hands to torch.tensor (each camera's point list, in the reference's order) and
which init files it saves.  Only this generator reads the reference.

Scenes:
  aachen_generic, dubrovnik_generic: random poses, landscape and portrait images, points crowded into a few cells, some
    off the image and behind the camera; every projection is kept >= 1e-3 px from a cell edge and depths in one cell
    >= 1e-4 apart (relative), so that any float32 summation order gives the same maps.
  dubrovnik_exact: axis-aligned poses, integer translations, small-integer and dyadic points, a power-of-two focal length
    and scale, so that every pose product is exact: equal-depth ties, duplicate observations, points behind the camera,
    off-image clamps, depth-0 points in the corners (after a nearer, before a farther, and after a negative depth), a
    camera without observations (skipped: empty z-buffer), an ignored and a missing image.

    python tests/golden/make_render_golden.py      (needs cv2 and the reference checkout)
"""
from __future__ import annotations

import ast
import math
import os
import sys
import tempfile
from pathlib import Path

import cv2
import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
OUT = Path(__file__).resolve().parent / "render"
sys.path.insert(0, str(ROOT))

from esac_b200.prepare import camera_geometry  # noqa: E402


def find_reference() -> Path:
    if os.environ.get("ESAC_REFERENCE"):
        return Path(os.environ["ESAC_REFERENCE"])
    for d in ROOT.parents:
        if (d / "reference" / "datasets").is_dir():
            return d / "reference"
    raise SystemExit("no reference checkout: set ESAC_REFERENCE")


def load_function(script: Path, name: str, globs: dict):
    tree = ast.parse(script.read_text())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), str(script), "exec"), globs)
    return globs[name]


class OsProxy:
    system = staticmethod(lambda cmd: 0)

    def __getattr__(self, k):
        return getattr(os, k)


class TorchProxy:
    def __init__(self):
        self.tensor_lists, self.saved = [], []

    def tensor(self, data, *a, **k):
        if isinstance(data, list):
            self.tensor_lists.append(data)
        return torch.tensor(data, *a, **k)

    def save(self, obj, path):
        self.saved.append(os.path.basename(path))
        torch.save(obj, path)

    def __getattr__(self, k):
        return getattr(torch, k)


def mkdir(d):
    os.makedirs(d, exist_ok=True)


def rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    if q[0] < 0:
        q = -q
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return q, R


def project64(pose32, X32, f, s, h, w):
    """u, v, z in float64 from the float32 pose and point (the margins below are far wider than any float32 rounding)."""
    cam = pose32[:3, :3].astype(np.float64) @ X32.astype(np.float64) + pose32[:3, 3].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = cam[0] * np.float64(np.float32(f)) / cam[2] * np.float64(np.float32(s)) + w / 2
        v = cam[1] * np.float64(np.float32(f)) / cam[2] * np.float64(np.float32(s)) + h / 2
    return u, v, cam[2]


def keep_margins(obs, poses, pts, cams):
    """Drops points (all their observations) whose projection is < 1e-3 px from a cell edge, or whose depth is within
    1e-4 (relative) of another point's in the same cell of the same camera."""
    alive = np.ones(len(pts), bool)
    for _ in range(10):
        cells = {}
        for c, j in obs:
            if not alive[j]:
                continue
            f, s, h, w = cams[c]
            u, v, z = project64(poses[c], pts[j], f, s, h, w)
            for q in (u, v):
                if abs(q) < 1e6 and abs(q - round(q)) < 1e-3:
                    alive[j] = False
            if alive[j]:
                cell = (c, int(min(max(v, 0), h - 1)), int(min(max(u, 0), w - 1)))
                cells.setdefault(cell, []).append((z, j))
        changed = False
        for lst in cells.values():
            for a in range(len(lst)):
                for b in range(a + 1, len(lst)):
                    (za, ja), (zb, jb) = lst[a], lst[b]
                    if ja != jb and alive[ja] and alive[jb] and abs(za - zb) < 1e-4 * max(abs(za), abs(zb)):
                        alive[jb] = False
                        changed = True
        if not changed:
            break
    return alive


def generic_points(rng, poses, cams, n_home=50):
    """Points made in each camera's frame (crowded cells, off-image, behind), each also listed by 0-2 other cameras."""
    pts, obs = [], []
    C = len(poses)
    for c in range(C):
        f, s, h, w = cams[c]
        R, t = poses[c][:3, :3].astype(np.float64), poses[c][:3, 3].astype(np.float64)
        for k in range(n_home):
            kind = rng.random()
            if kind < 0.6:   # crowded into a few cells
                u, v = w / 2 + rng.normal(0, 1.5), h / 2 + rng.normal(0, 1.5)
            elif kind < 0.8:
                u, v = rng.uniform(0, w), rng.uniform(0, h)
            else:            # off the image
                u, v = rng.uniform(-2 * w, 3 * w), rng.uniform(-2 * h, 3 * h)
            d = rng.uniform(2, 20) * (-1 if rng.random() < 0.1 else 1)
            camp = np.array([(u - w / 2) / s / f * d, (v - h / 2) / s / f * d, d])
            X = R.T @ (camp - t)
            j = len(pts)
            pts.append(X)
            viewers = [c] + list(rng.choice(C, int(rng.integers(0, 3)), replace=True))
            rng.shuffle(viewers)
            obs.extend((int(v_), j) for v_ in viewers)
    return np.array(pts), obs


def fmt(x):
    return repr(float(x))


# ---- Aachen ---------------------------------------------------------------------------------------------------------
AACHEN_IMAGES = [("db/1001.jpg", (60, 80)), ("db/1002.jpg", (80, 60)), ("db/1003.jpg", (683, 1024)),
                 ("db/1004.jpg", (1024, 683)), ("db/1005.jpg", (45, 80)), ("db/1006.jpg", (60, 80)),
                 ("db/9999.jpg", (60, 80))]   # the last is in the NVM, not in the db list


def aachen_generic(rng):
    C = len(AACHEN_IMAGES)
    poses, quats, centres, focals, cams = [], [], [], [], []
    for name, (h, w) in AACHEN_IMAGES:
        q, R = rotation(rng)
        Cw = rng.uniform(-10, 10, 3)
        f = float(rng.uniform(0.8, 1.3) * max(h, w))
        quats.append(q)
        centres.append(Cw)
        focals.append(f)
        pose = np.eye(4)
        pose[:3, :3] = R
        pose[:3, 3] = -R @ Cw
        poses.append(pose.astype(np.float32))
        oh, ow, osc, _ = camera_geometry("aachen", h, w)
        cams.append((f, osc, oh, ow))
    pts, obs = generic_points(rng, poses, cams)
    pts32 = pts.astype(np.float32)
    alive = keep_margins(obs, poses, pts32, cams)
    keep = np.flatnonzero(alive)
    lines = ["NVM_V3", "", str(C)]
    for (name, _), q, Cw, f in zip(AACHEN_IMAGES, quats, centres, focals):
        lines.append(" ".join([name, fmt(f)] + [fmt(v) for v in q] + [fmt(v) for v in Cw] + [fmt(rng.uniform(-0.1, 0.1)), "0"]))
    lines += ["", str(len(keep))]
    for j in keep:
        views = [c for c, jj in obs if jj == j]
        toks = [fmt(v) for v in pts32[j]] + ["128", "128", "128", str(len(views))]
        for c in views:
            toks += [str(c), str(int(rng.integers(0, 9999))), "0.5", "-0.5"]
        lines.append(" ".join(toks))
    lines += ["", "0", ""]
    nvm = "\n".join(lines) + "\n"
    db = "".join(f"{n} SIMPLE_RADIAL 1 2 3\n" for n, _ in AACHEN_IMAGES[:-1])
    return nvm, db


def run_aachen(ref: Path, nvm: str, db: str, tmp: Path):
    src = tmp / "src"
    (src / "images" / "db").mkdir(parents=True)
    (src / "recon.nvm").write_text(nvm)
    (src / "db.list.txt").write_text(db)
    for name, (h, w) in AACHEN_IMAGES:
        cv2.imwrite(str(src / "images" / name), np.zeros((h, w, 3), np.uint8))
    tp = TorchProxy()
    g = {"os": OsProxy(), "torch": tp, "math": math, "np": np, "cv": cv2, "recon_file": "recon.nvm",
         "image_folder": "images/", "dst_folder": "dst", "mkdir": mkdir, "mode": "training", "print": lambda *a: None}
    fn = load_function(ref / "datasets" / "setup_aachen.py", "create_training_set", g)
    cwd = os.getcwd()
    os.chdir(src)
    try:
        fn("db.list.txt")
    finally:
        os.chdir(cwd)
    return tp, tmp / "dst" / "training"


# ---- Dubrovnik ------------------------------------------------------------------------------------------------------
def bundle_text(poses, focals, pts32, obs, rng):
    """Bundler v0.3: the world -> camera pose P is written as R = diag(1,-1,-1) P_R, t = diag(1,-1,-1) P_t."""
    C = len(poses)
    lines = ["# Bundle file v0.3", f"{C} {len(pts32)}"]
    flip = np.array([1.0, -1.0, -1.0])
    for P, f in zip(poses, focals):
        lines.append(f"{fmt(f)} 0 0")
        for r in range(3):
            lines.append(" ".join(fmt(flip[r] * P[r, k]) for k in range(3)))
        lines.append(" ".join(fmt(flip[r] * P[r, 3]) for r in range(3)))
    for j, X in enumerate(pts32):
        views = [c for c, jj in obs if jj == j]
        lines.append(" ".join(fmt(v) for v in X))
        lines.append("128 128 128")
        lines.append(" ".join([str(len(views))] + sum(([str(c), str(int(rng.integers(0, 9999))), "0.25", "-0.75"]
                                                       for c in views), [])))
    return "\n".join(lines) + "\n"


def dubrovnik_generic(rng):
    images = [("a_1.jpg", (60, 80)), ("b_2.jpg", (80, 60)), ("c_3.jpg", (683, 1024)), ("d_4.jpg", (1024, 683)),
              ("e_5.jpg", (36, 64))]
    poses, focals, cams = [], [], []
    for name, (h, w) in images:
        _, R = rotation(rng)
        t = rng.uniform(-5, 5, 3)
        P = np.eye(4)
        P[:3, :3] = R
        P[:3, 3] = t
        f = float(rng.uniform(0.8, 1.3) * max(h, w))
        poses.append(P.astype(np.float32))
        focals.append(f)
        oh, ow, osc, _ = camera_geometry("dubrovnik", h, w)
        cams.append((f, osc, oh, ow))
    pts, obs = generic_points(rng, poses, cams)
    pts32 = pts.astype(np.float32)
    alive = keep_margins(obs, poses, pts32, cams)
    keep = np.flatnonzero(alive)
    remap = {int(j): i for i, j in enumerate(keep)}
    obs = [(c, remap[j]) for c, j in obs if alive[j]]
    text = bundle_text(poses, focals, pts32[keep], obs, rng)
    # list.db.txt in an order of its own: the cameras come out in the list's order
    order = [2, 0, 4, 1, 3]
    listing = "".join(f"db/{images[c][0]}\n" for c in order)
    return text, listing, images, set(n for n, _ in images)


def dubrovnik_exact():
    """Exact arithmetic: f = 64, out scale 0.5 (160 x 120 images -> 80 x 60 maps, 120 x 160 -> 60 x 80)."""
    images = [("x_1.jpg", (120, 160)), ("y_2.jpg", (160, 120)), ("z_3.jpg", (120, 160)), ("westius_2275531184.jpg", (120, 160)),
              ("gone_5.jpg", (120, 160)), ("w_6.jpg", (160, 120))]
    P0 = np.eye(4, dtype=np.float32)
    P1 = np.array([[0, 1, 0, 1], [-1, 0, 0, 0], [0, 0, 1, 2], [0, 0, 0, 1]], np.float32)
    P2 = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]], np.float32)   # everything behind
    poses = [P0, P1, P2, P0, P0, P0]
    focals = [64.0] * 6
    pts, obs = [], []

    def add(X, cams):
        pts.append(X)
        obs.extend((c, len(pts) - 1) for c in cams)

    # camera 0 (80 x 60): u = 32 x / z + 40, v = 32 y / z + 30
    add((1, 1, 8), [0])                 # cell (34, 44), depth 8
    add((0.5, 0.5, 4), [0, 0])          # the same cell, nearer; observed twice
    add((0.25, 0.25, 2), [0])           # the same cell, nearer still
    add((-0.5, -0.5, -4), [0])          # the same cell, behind the camera: a negative depth beats them all
    add((0.0625, 0.0625, 4), [0])       # u = v - 10 = 40.5: cell (30, 40), depth 4
    add((0, 0, 4), [0, 1])              # the same cell and depth: the earlier point stays
    add((0.5, 0.5, -2), [0])            # behind the camera, projected onto the image: cell (22, 32)
    add((1, 2, -2), [0])                # behind: v = -2, clamped onto row 0
    add((10, 10, 1), [0, 1])            # off the image: corner (59, 79), depth 1
    add((3, 3, 0), [0])                 # depth 0, u = v = +inf: the same corner, written over the depth 1
    add((50, 50, 6), [0])               # after the depth 0: written whatever its depth
    add((-5, -5, 0), [0])               # depth 0 alone in corner (0, 0)
    add((-7, 9, 0), [0])                # depth 0 in corner (59, 0)
    add((-20, 30, -1), [0])             # behind: u = 680, v = -930, corner (0, 79), negative depth
    add((9, -9, 0), [0])                # depth 0 in corner (0, 79) after the negative depth: not written
    add((20, -30, 3), [0])              # corner (0, 79), positive: loses to the negative depth
    add((-9, 9, 0), [0])                # a second depth 0 in corner (59, 0): the last one stays
    # camera 1 (60 x 80, cam = (y + 1, -x, z + 2)): u = 32 cam.x / cam.z + 30, v = 32 cam.y / cam.z + 40
    add((2, 0.5, 2), [1])               # cell (24, 42), depth 4
    add((2, 0.5, 2), [1])               # an identical point: a tie at the same depth, the first stays
    add((3, 5, -2), [1])                # cam = (6, -3, 0): corner (0, 59), written over the depth 3 of (10, 10, 1)
    # camera 2: every point behind (P2 flips z)
    add((1, 1, 3), [2])
    add((-2, 1, 5), [2, 2])
    # camera 3 (ignored image), 4 (missing image): listed, never written
    add((1, 1, 3), [3, 4])
    # camera 5: no observation -> empty z-buffer, skipped.  (Camera 0's depths sum to 1, not 0: the reference tests the
    # sum, which exact cancellation would also zero.)
    pts32 = np.array(pts, np.float32)
    rng = np.random.default_rng(0)
    text = bundle_text(poses, focals, pts32, obs, rng)
    listing = "".join(f"db/{n}\n" for n, _ in images)
    existing = set(n for n, _ in images) - {"gone_5.jpg"}
    return text, listing, images, existing


def run_dubrovnik(ref: Path, text: str, listing: str, images, existing, tmp: Path):
    src = tmp / "src"
    src.mkdir(parents=True)
    db = tmp / "dbimages"
    db.mkdir()
    (src / "bundle.out").write_text(text)
    (src / "list.db.txt").write_text(listing)
    for name, (h, w) in images:
        if name in existing:
            cv2.imwrite(str(db / name), np.zeros((h, w, 3), np.uint8))
    tp = TorchProxy()

    class Opt:
        dbfolder = "dbimages"
    ignore = ["klazien_2867455427.jpg", "eas8302_2799908943.jpg", "28512365@N08_2967791490.jpg",
              "neozeitgeist_2614406528.jpg", "22417886@N02_2162265990.jpg", "westius_2275531184.jpg"]
    g = {"os": OsProxy(), "torch": tp, "math": math, "cv2": cv2, "dst_folder": "dst", "mkdir": mkdir, "opt": Opt,
         "existing_images": os.listdir(db), "ignore_images": ignore, "print": lambda *a: None}
    fn = load_function(ref / "datasets" / "setup_dubrovnik.py", "create_set", g)
    cwd = os.getcwd()
    os.chdir(src)
    try:
        fn("bundle.out", "list.db.txt", "list.db.txt", training=True)
    finally:
        os.chdir(cwd)
    # the reference passes each camera's pose list to torch.tensor before its point list
    tp.tensor_lists = tp.tensor_lists[1::2]
    return tp, tmp / "dst" / "training"


def collect(tp: TorchProxy, dst: Path, kind: str, recon: str, listing: str, images, existing):
    saved = [n[:-4] for n in tp.saved]
    maps = [torch.load(dst / "init" / (n + ".dat")).numpy() for n in saved]
    poses = np.array([[float(v) for v in (dst / "poses" / (n + ".txt")).read_text().split()] for n in saved]).reshape(-1, 4, 4)
    calib = [(dst / "calibration" / (n + ".txt")).read_text() for n in saved]
    cam_pts = [np.asarray(lst, np.float32).reshape(-1, 4)[:, :3] for lst in tp.tensor_lists]
    return dict(
        kind=np.array(kind), recon=np.array(recon), listing=np.array(listing),
        image_names=np.array([n for n, _ in images]), image_hw=np.array([hw for _, hw in images], np.int64),
        existing=np.array(sorted(existing)), saved=np.array(saved),
        map_shapes=np.array([m.shape[1:] for m in maps], np.int64),
        maps=np.concatenate([m.reshape(-1) for m in maps]).astype(np.float32),
        poses=poses, calib=np.array(calib),
        cam_counts=np.array([len(p) for p in cam_pts], np.int64),
        cam_points=np.concatenate(cam_pts).astype(np.float32) if cam_pts else np.zeros((0, 3), np.float32))


def main():
    ref = find_reference()
    OUT.mkdir(exist_ok=True)
    rng = np.random.default_rng(20261017)
    with tempfile.TemporaryDirectory() as d:
        nvm, db = aachen_generic(rng)
        tp, dst = run_aachen(ref, nvm, db, Path(d) / "aachen")
        np.savez_compressed(OUT / "aachen_generic.npz",
                            **collect(tp, dst, "aachen", nvm, db, AACHEN_IMAGES, [n for n, _ in AACHEN_IMAGES]))
        text, listing, images, existing = dubrovnik_generic(rng)
        tp, dst = run_dubrovnik(ref, text, listing, images, existing, Path(d) / "dub")
        np.savez_compressed(OUT / "dubrovnik_generic.npz", **collect(tp, dst, "dubrovnik", text, listing, images, existing))
        text, listing, images, existing = dubrovnik_exact()
        tp, dst = run_dubrovnik(ref, text, listing, images, existing, Path(d) / "exact")
        np.savez_compressed(OUT / "dubrovnik_exact.npz", **collect(tp, dst, "dubrovnik", text, listing, images, existing))
    for p in sorted(OUT.glob("*.npz")):
        z = np.load(p)
        print(p.name, "cameras written:", list(z["saved"]), "observations:", int(z["cam_counts"].sum()), f"{p.stat().st_size} B")


if __name__ == "__main__":
    main()
