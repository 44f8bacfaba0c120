"""The training sets of Aachen and Dubrovnik from their SfM reconstructions: ground-truth scene-coordinate maps
(init/<name>.dat), poses (poses/<name>.txt) and calibration (calibration/<name>.txt) as the reference's converters write
them (datasets/setup_aachen.py:56-212 create_training_set, datasets/setup_dubrovnik.py:54-207 create_set), with the
z-buffer render on the GPU (api.render_init_maps) instead of a Python loop over every observation.

    rec = read_nvm("aachen_cvpr2018_db.nvm", "aachen_cvpr2018_db.list.txt")
    sizes = image_sizes([image_folder + n for n in rec.images])
    out = write_training_set("aachen/training", rec, sizes)
    cluster_environment(out.maps, num_clusters=...)

    python -m esac_b200.prepare aachen --nvm aachen_cvpr2018_db.nvm --list aachen_cvpr2018_db.list.txt \
        --images images_upright/ --out aachen/training
    python -m esac_b200.prepare dubrovnik --bundle Dubrovnik6K/bundle/bundle.db.out --list Dubrovnik6K/list.db.txt \
        --images dubrovnik_db_images/ --out dubrovnik/training

Each reader builds the observations as the reference does: one list per camera, in the order of the points in the file
(a point that lists a camera twice is observed twice), and the cameras in the order the reference visits them.  The
renderer evaluates each projection in one stated float32 order; the reference's torch.mm may differ from it by an ulp, so
a cell can differ where a projection lies within a few ulps of a cell edge or two depths within a few ulps of each other.

Not covered here, and left to the setup scripts: the downloads, the rgb side (Aachen's cv.undistort + cv.resize, the image
links), and the test sets (query poses and calibration, no init maps).
"""
from __future__ import annotations

import argparse
import math
import os
from dataclasses import dataclass

import numpy as np

# setup_dubrovnik.py:46-52: outlier training images
DUBROVNIK_IGNORE = ("klazien_2867455427.jpg", "eas8302_2799908943.jpg", "28512365@N08_2967791490.jpg",
                    "neozeitgeist_2614406528.jpg", "22417886@N02_2162265990.jpg", "westius_2275531184.jpg")


@dataclass
class Reconstruction:
    kind: str                # "aachen" or "dubrovnik": the output size rule and the calibration written
    names: list              # output file name of each camera (Aachen: the image path with '/' -> '_')
    images: list             # each camera's image, relative to the image folder
    points: np.ndarray       # float32 [P,3]
    offsets: np.ndarray      # int64 [C+1]: camera c observes indices[offsets[c]:offsets[c+1]]
    indices: np.ndarray      # int32 [V] point of each observation, in file order
    poses: np.ndarray        # float32 [C,4,4] world -> camera
    focal: np.ndarray        # float64 [C] the reconstruction's focal length


def _csr(cam_of_obs: list, pt_of_obs: list, cameras: list) -> tuple:
    """Observations (camera in the file, point) in file order -> the CSR of the chosen cameras, in their order."""
    cam = np.asarray(cam_of_obs, np.int64)
    pt = np.asarray(pt_of_obs, np.int32)
    order = np.argsort(cam, kind="stable")
    cam_s, pt_s = cam[order], pt[order]
    starts = np.searchsorted(cam_s, np.asarray(cameras, np.int64), "left")
    ends = np.searchsorted(cam_s, np.asarray(cameras, np.int64), "right")
    counts = ends - starts
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    indices = np.concatenate([pt_s[a:b] for a, b in zip(starts, ends)]) if len(cameras) else np.zeros(0, np.int32)
    return offsets, indices.astype(np.int32)


def _rodrigues(r: np.ndarray) -> np.ndarray:
    """cv::Rodrigues of a rotation vector, float64, in OpenCV's op order (c I + (1 - c) r r^T + s [r]x)."""
    theta = math.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
    if theta < np.finfo(np.float64).eps:
        return np.eye(3)
    c, s = math.cos(theta), math.sin(theta)
    c1 = 1.0 - c
    itheta = 1.0 / theta
    x, y, z = r[0] * itheta, r[1] * itheta, r[2] * itheta
    rrt = np.array([[x * x, x * y, x * z], [x * y, y * y, y * z], [x * z, y * z, z * z]])
    rx = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]], np.float64)
    return c * np.eye(3) + c1 * rrt + s * rx


def _nvm_pose(camera: list) -> np.ndarray:
    """setup_aachen.py:116-138: quaternion -> axis-angle -> Rodrigues, t = -R C, as float32 [4,4]."""
    w, qx, qy, qz = (float(v) for v in camera[2:6])
    angle = 2 * math.acos(w)
    n = math.sqrt(1 - w ** 2)
    R = _rodrigues(np.array([qx / n * angle, qy / n * angle, qz / n * angle]))
    C = np.array([[float(v)] for v in camera[6:9]])
    t = -np.matmul(R, C)
    pose = np.concatenate((np.concatenate((R, t), axis=1), [[0, 0, 0, 1]]), axis=0)
    return pose.astype(np.float32)


def read_nvm(nvm_file: str, list_file: str) -> Reconstruction:
    """Aachen (setup_aachen.py:56-138): the NVM cameras listed in list_file, in NVM order.  As in the reference, a camera's
    pose and focal length come from the NVM camera at the position its image has in list_file (the same camera when the
    list follows the NVM's order), and its points from its own position in the NVM."""
    with open(nvm_file) as f:
        rec = f.readlines()
    with open(list_file) as f:
        image_list = [line.split()[0] for line in f.readlines()]
    position = {}
    for i, name in enumerate(image_list):
        position.setdefault(name, i)
    num_cams = int(rec[2])
    num_pts = int(rec[num_cams + 4])
    cameras = [c.split() for c in rec[3:3 + num_cams]]
    points = np.empty((num_pts, 3), np.float32)
    cam_of_obs, pt_of_obs = [], []
    start = num_cams + 5
    for j in range(num_pts):
        tok = rec[start + j].split()
        points[j] = [float(x) for x in tok[0:3]]
        views = int(tok[6])
        cams = [int(tok[7 + k * 4]) for k in range(views)]
        cam_of_obs.extend(cams)
        pt_of_obs.extend([j] * views)
    chosen, names, images, poses, focal = [], [], [], [], []
    for cam_idx in range(num_cams):
        image = cameras[cam_idx][0]
        if image not in position:
            continue
        camera = cameras[position[image]]
        chosen.append(cam_idx)
        images.append(image)
        names.append(image.replace("/", "_"))
        poses.append(_nvm_pose(camera))
        focal.append(float(camera[1]))
    offsets, indices = _csr(cam_of_obs, pt_of_obs, chosen)
    return Reconstruction("aachen", names, images, points, offsets, indices,
                          np.asarray(poses, np.float32).reshape(-1, 4, 4), np.asarray(focal, np.float64))


def read_bundler(bundle_file: str, list_file: str, existing=None, ignore=DUBROVNIK_IGNORE) -> Reconstruction:
    """Dubrovnik (setup_dubrovnik.py:54-147, training): the cameras of list_file in its order, each mapped to the bundle
    camera at the first line of list_file equal to it, named without its first three characters ("db/"), skipped when
    that name is not in `existing` (the database folder's file names; None: all exist) or is in `ignore`."""
    with open(bundle_file) as f:
        rec = f.readlines()
    with open(list_file) as f:
        lines = f.readlines()
    stripped = {}
    for i, line in enumerate(lines):
        stripped.setdefault(line.strip(), i)
    num_cams, num_pts = (int(v) for v in rec[1].split()[:2])
    existing = None if existing is None else set(existing)
    points = np.empty((num_pts, 3), np.float32)
    cam_of_obs, pt_of_obs = [], []
    start = 2 + num_cams * 5
    for j in range(num_pts):
        points[j] = [float(x) for x in rec[start + 3 * j].split()]
        tok = rec[start + 3 * j + 2].split()
        views = int(tok[0])
        cam_of_obs.extend(int(tok[1 + k * 4]) for k in range(views))
        pt_of_obs.extend([j] * views)
    chosen, names, poses, focal = [], [], [], []
    for line in lines:
        image_file = line.split()[0]
        cam_idx = stripped[image_file]
        name = image_file[3:]
        if (existing is not None and name not in existing) or name in ignore:
            continue
        rows = [[float(x) for x in rec[3 + cam_idx * 5 + k].split()] for k in range(3)]
        t = [float(x) for x in rec[6 + cam_idx * 5].split()]
        pose = [rows[0] + [t[0]], [-x for x in rows[1]] + [-t[1]], [-x for x in rows[2]] + [-t[2]], [0.0, 0.0, 0.0, 1.0]]
        chosen.append(cam_idx)
        names.append(name)
        poses.append(np.asarray(pose, np.float64).astype(np.float32))
        focal.append(float(rec[2 + cam_idx * 5].split()[0]))
    offsets, indices = _csr(cam_of_obs, pt_of_obs, chosen)
    return Reconstruction("dubrovnik", names, list(names), points, offsets, indices,
                          np.asarray(poses, np.float32).reshape(-1, 4, 4), np.asarray(focal, np.float64))


def camera_geometry(kind: str, height: int, width: int) -> tuple:
    """(out_h, out_w, out_scale, img_scale) of an image of height x width.  Aachen (setup_aachen.py:146-164): the short
    side to 480 px, then out = ceil(img / 8); Dubrovnik (setup_dubrovnik.py:155-167): the short side straight to 60
    cells.  img_scale (Aachen's calibration factor) is 1 for Dubrovnik."""
    aspect = height / width
    if kind == "aachen":
        if aspect > 1:
            img_w, img_h = 480, int(math.ceil(480 * aspect))
        else:
            img_w, img_h = int(math.ceil(480 / aspect)), 480
        out_w, out_h = int(math.ceil(img_w / 8)), int(math.ceil(img_h / 8))
        return out_h, out_w, out_w / width, img_w / width
    if kind == "dubrovnik":
        if aspect > 1:
            out_w, out_h = 60, int(math.ceil(60 * aspect))
        else:
            out_w, out_h = int(math.ceil(60 / aspect)), 60
        return out_h, out_w, out_w / width, 1.0
    raise ValueError(f"unknown reconstruction kind {kind!r}")


def image_sizes(paths) -> list:
    """(height, width) of each image from its header, as cv2.imread sees it (EXIF orientations 5-8 swap the sides)."""
    from PIL import Image
    out = []
    for p in paths:
        with Image.open(p) as im:
            w, h = im.size
            if im.getexif().get(0x0112, 1) in (5, 6, 7, 8):
                w, h = h, w
        out.append((h, w))
    return out


@dataclass
class TrainingSet:
    names: list    # the cameras written, in order
    skipped: list  # the cameras skipped (Dubrovnik: every z-buffer cell 0)
    maps: list     # float32 [3,h,w] CUDA views of every rendered camera, written or not
    counts: object  # int32 [C] cells written per camera


def _pose_text(pose: np.ndarray) -> str:
    import torch
    inv = torch.from_numpy(np.ascontiguousarray(pose, np.float32)).inverse()
    return "".join(" ".join(str(float(inv[r, c])) for c in range(4)) + "\n" for r in range(4))


def write_training_set(dst: str, rec: Reconstruction, sizes) -> TrainingSet:
    """Renders every camera of `rec` on the GPU (sizes: its image's (height, width), in rec's order) and writes its files
    under dst (save_training_files).  Dubrovnik skips a camera whose z-buffer is 0 in every cell; the reference tests the
    float32 sum of the z-buffer, which is also 0 when depths cancel exactly: such a camera is written here."""
    from . import api
    C = len(rec.names)
    if len(sizes) != C:
        raise RuntimeError(f"write_training_set: {len(sizes)} image sizes for {C} cameras")
    geo = [camera_geometry(rec.kind, int(h), int(w)) for h, w in sizes]
    shapes = np.array([[g[0], g[1]] for g in geo], np.int64)
    maps, counts, zbufs = api.render_init_maps(rec.points, rec.offsets, rec.indices, rec.poses, rec.focal,
                                               [g[2] for g in geo], shapes, zbuffer=rec.kind == "dubrovnik")
    import torch
    empty = [False] * C
    if zbufs is not None:
        empty = torch.stack([(z != 0).any() for z in zbufs]).logical_not().cpu().tolist()
    written, skipped = save_training_files(dst, rec, sizes, maps, empty)
    return TrainingSet(written, skipped, maps, counts)


def save_training_files(dst: str, rec: Reconstruction, sizes, maps, empty) -> tuple:
    """Writes, under dst, for each camera c of `rec` with empty[c] false: init/<name[:-4]>.dat (torch.save of a CPU
    float32 [3,h,w] copy of maps[c], which may be a view of a larger buffer), poses/<name[:-3]>txt (the float32 inverse
    of the pose, camera -> world, four lines of str(float)) and calibration/<name[:-3]>txt (str of the focal length times
    img_scale for Aachen, of the focal length for Dubrovnik).  Returns (names written, names skipped)."""
    import torch
    for sub in ("init", "poses", "calibration"):
        os.makedirs(os.path.join(dst, sub), exist_ok=True)
    written, skipped = [], []
    for c, name in enumerate(rec.names):
        if empty[c]:
            skipped.append(name)
            continue
        # a copy of the map alone: saving a view would save the whole buffer it lives in
        m = torch.as_tensor(maps[c]).to("cpu", copy=True)
        torch.save(m, os.path.join(dst, "init", name[:-4] + ".dat"))
        h, w = sizes[c]
        calib = rec.focal[c] * camera_geometry(rec.kind, int(h), int(w))[3] if rec.kind == "aachen" else rec.focal[c]
        with open(os.path.join(dst, "calibration", name[:-3] + "txt"), "w") as f:
            f.write(str(float(calib)))
        with open(os.path.join(dst, "poses", name[:-3] + "txt"), "w") as f:
            f.write(_pose_text(rec.poses[c]))
        written.append(name)
    return written, skipped


def main(argv=None):
    ap = argparse.ArgumentParser(description="Write the init maps, poses and calibration of Aachen's or Dubrovnik's "
                                             "training set from its SfM reconstruction, rendered on the GPU.")
    ap.add_argument("kind", choices=("aachen", "dubrovnik"))
    ap.add_argument("--nvm", help="aachen: aachen_cvpr2018_db.nvm")
    ap.add_argument("--bundle", help="dubrovnik: Dubrovnik6K/bundle/bundle.db.out")
    ap.add_argument("--list", required=True, help="aachen_cvpr2018_db.list.txt or Dubrovnik6K/list.db.txt")
    ap.add_argument("--images", required=True, help="the image folder (aachen: images_upright/, dubrovnik: the db images)")
    ap.add_argument("--out", required=True, help="the training folder to write, e.g. aachen/training")
    a = ap.parse_args(argv)
    if a.kind == "aachen":
        if not a.nvm:
            ap.error("aachen needs --nvm")
        rec = read_nvm(a.nvm, a.list)
    else:
        if not a.bundle:
            ap.error("dubrovnik needs --bundle")
        rec = read_bundler(a.bundle, a.list, existing=os.listdir(a.images))
    sizes = image_sizes([os.path.join(a.images, n) for n in rec.images])
    out = write_training_set(a.out, rec, sizes)
    print(f"{len(out.names)} cameras written, {len(out.skipped)} skipped (empty z-buffer), "
          f"{int(rec.offsets[-1])} observations of {len(rec.points)} points")


if __name__ == "__main__":
    main()
