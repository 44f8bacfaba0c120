"""Restatements of the init-map renderer (esac_b200/csrc/render.cu, api.render_init_maps) for the tests.

render_fixed: a vectorised numpy float32 restatement of the kernel, bit for bit: each pose row in the order
((r0 x + r1 y) + r2 z) + r3, u = ((cam.x f) / cam.z) s + w/2, every op rounded to float32; then per cell the rule the
reference's serial z-test (`zbuf == 0 or zbuf > z`, setup_aachen.py:184-202, setup_dubrovnik.py:171-190) amounts to: the
nearest non-zero depth, earliest on a tie, after the last written depth-0 point (the last one before the cell's first
negative depth), else that point, else nothing.

render_serial: the reference's loop itself, one observation at a time with torch ops, with a pluggable 4x4 . 4x1 product:
"torch" (torch.mm, the reference's) or "fixed" (the kernel's order).  With "fixed" it equals render_fixed bitwise, which
holds the restated cell rule to the plain loop.

Both take the arguments of api.render_init_maps as numpy / torch CPU data: points float32 [P,3], offsets int [C+1],
indices int [V], poses [C,4,4] or [C,3,4], focal [C], out_scale [C], shapes [(h, w)] * C.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def _np(t, dtype=None):
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=dtype)


def _poses34(poses) -> np.ndarray:
    p = _np(poses, F32)
    return np.ascontiguousarray(p[:, :3, :])


def fixed_product(pose34: np.ndarray, X: np.ndarray) -> np.ndarray:
    """cam = pose . [x, y, z, 1] row by row in the kernel's float32 order; X float32 [..., 3] -> [..., 3]."""
    x, y, z = X[..., 0], X[..., 1], X[..., 2]
    r = pose34.astype(F32)
    rows = [((r[..., i, 0] * x + r[..., i, 1] * y) + r[..., i, 2] * z) + r[..., i, 3] for i in range(3)]
    return np.stack(rows, -1).astype(F32)


def render_fixed(points, offsets, indices, poses, focal, out_scale, shapes):
    """Returns (maps [list of float32 [3,h,w]], zbufs [list of float32 [h,w]], counts int32 [C], status int32 [C]);
    status bit 1: a point index outside [0, P), bit 2: a NaN projection (those observations take no part)."""
    pts = _np(points, F32).reshape(-1, 3)
    offs = _np(offsets, np.int64)
    idx = _np(indices, np.int64)
    P34 = _poses34(poses)
    f = _np(focal, np.float64).astype(F32)
    s = _np(out_scale, np.float64).astype(F32)
    C = len(shapes)
    hs = np.array([h for h, _ in shapes], np.int64)
    ws = np.array([w for _, w in shapes], np.int64)
    cell0 = np.concatenate([[0], np.cumsum(hs * ws)])
    V = int(offs[-1])
    cam = np.repeat(np.arange(C), np.diff(offs))
    status = np.zeros(C, np.int32)
    bad = (idx < 0) | (idx >= len(pts))
    np.bitwise_or.at(status, cam[bad], 1)
    X = pts[np.where(bad, 0, idx)] if len(pts) else np.zeros((V, 3), F32)
    cp = fixed_product(P34[cam], X)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = ((cp[:, 0] * f[cam]) / cp[:, 2]) * s[cam] + (ws[cam] / 2).astype(F32)
        v = ((cp[:, 1] * f[cam]) / cp[:, 2]) * s[cam] + (hs[cam] / 2).astype(F32)
    nan = ~bad & (np.isnan(u) | np.isnan(v))
    np.bitwise_or.at(status, cam[nan], 2)
    ok = ~bad & ~nan
    col = np.minimum(np.maximum(u[ok], F32(0)), (ws[cam[ok]] - 1).astype(F32)).astype(np.int64)
    row = np.minimum(np.maximum(v[ok], F32(0)), (hs[cam[ok]] - 1).astype(F32)).astype(np.int64)
    obs = np.flatnonzero(ok)
    cell = cell0[cam[ok]] + row * ws[cam[ok]] + col
    z = cp[ok, 2]
    ncell = int(cell0[-1])
    first_neg = np.full(ncell, V, np.int64)
    neg = z < 0
    np.minimum.at(first_neg, cell[neg], obs[neg])
    last_zero = np.full(ncell, -1, np.int64)
    zero = (z == 0) & (obs < first_neg[cell])
    np.maximum.at(last_zero, cell[zero], obs[zero])
    winner = last_zero.copy()
    near = (z != 0) & (obs > last_zero[cell])
    c_n, z_n, o_n = cell[near], z[near], obs[near]
    order = np.lexsort((o_n, z_n, c_n))
    c_s = c_n[order]
    first = np.ones(len(c_s), bool)
    first[1:] = c_s[1:] != c_s[:-1]
    winner[c_s[first]] = o_n[order][first]
    z_of = np.zeros(V, F32)
    z_of[obs] = z
    has = winner >= 0
    flat = np.zeros((ncell, 3), F32)
    flat[has] = pts[idx[winner[has]]]
    zflat = np.zeros(ncell, F32)
    zflat[has] = z_of[winner[has]]
    maps, zbufs = [], []
    counts = np.zeros(C, np.int32)
    for c in range(C):
        a, b = int(cell0[c]), int(cell0[c + 1])
        maps.append(np.ascontiguousarray(flat[a:b].T.reshape(3, int(hs[c]), int(ws[c]))))
        zbufs.append(zflat[a:b].reshape(int(hs[c]), int(ws[c])))
        counts[c] = int(has[a:b].sum())
    return maps, zbufs, counts, status


def render_serial(points, offsets, indices, poses, focal, out_scale, shapes, product: str = "torch"):
    """The reference's per-observation loop (one camera after the other); focal and out_scale are used as Python floats
    as the reference uses them.  Returns (maps, zbufs, counts) like render_fixed.  Raises as the reference does on a NaN
    projection (int(nan)) or an index out of range."""
    import torch
    pts = torch.as_tensor(_np(points, F32).reshape(-1, 3))
    offs = _np(offsets, np.int64)
    idx = _np(indices, np.int64)
    p = _np(poses, F32)
    if p.shape[1] == 3:
        p = np.concatenate([p, np.broadcast_to(np.array([0, 0, 0, 1], F32), (len(p), 1, 4))], 1)
    f = _np(focal, np.float64)
    s = _np(out_scale, np.float64)
    maps, zbufs, counts = [], [], []
    for c, (out_h, out_w) in enumerate(shapes):
        cam_pose = torch.as_tensor(np.ascontiguousarray(p[c]))
        focal_length, scale = float(f[c]), float(s[c])
        out_tensor = torch.zeros((3, out_h, out_w))
        out_zbuffer = torch.zeros((out_h, out_w))
        written = np.zeros((out_h, out_w), bool)
        for o in range(int(offs[c]), int(offs[c + 1])):
            X = pts[int(idx[o])]
            scene_pt = torch.cat([X, torch.ones(1)]).unsqueeze(0).transpose(0, 1)
            if product == "torch":
                cam_pt = torch.mm(cam_pose, scene_pt)
            else:
                cam_pt = torch.as_tensor(np.append(fixed_product(p[c][:3], X.numpy()), F32(1))).unsqueeze(1)
            img_pt = cam_pt[0:2, 0] * focal_length / cam_pt[2, 0] * scale
            y = img_pt[1] + out_h / 2
            x = img_pt[0] + out_w / 2
            x = int(torch.clamp(x, min=0, max=out_w - 1))
            y = int(torch.clamp(y, min=0, max=out_h - 1))
            if out_zbuffer[y, x] == 0 or out_zbuffer[y, x] > cam_pt[2, 0]:
                out_zbuffer[y, x] = cam_pt[2, 0]
                out_tensor[:, y, x] = X
                written[y, x] = True
        maps.append(out_tensor.numpy())
        zbufs.append(out_zbuffer.numpy())
        counts.append(int(written.sum()))
    return maps, zbufs, np.array(counts, np.int32)


def fixture_reconstruction(npz, tmp_dir):
    """A fixture of tests/golden/render/ (make_render_golden.py) read back through esac_b200.prepare's reader: returns
    (the fixture, the Reconstruction, the image sizes (h, w) in its camera order)."""
    import os

    from esac_b200 import prepare
    z = np.load(npz)
    kind = str(z["kind"])
    rec_path, list_path = os.path.join(tmp_dir, "recon.txt"), os.path.join(tmp_dir, "list.txt")
    with open(rec_path, "w") as f:
        f.write(str(z["recon"]))
    with open(list_path, "w") as f:
        f.write(str(z["listing"]))
    if kind == "aachen":
        rec = prepare.read_nvm(rec_path, list_path)
    else:
        rec = prepare.read_bundler(rec_path, list_path, existing=[str(n) for n in z["existing"]])
    hw = {str(n): tuple(int(v) for v in s) for n, s in zip(z["image_names"], z["image_hw"])}
    return z, rec, [hw[n] for n in rec.images]


def fixture_maps(z) -> list:
    """The reference's init maps of a fixture, in the order it saved them."""
    out, at = [], 0
    for h, w in z["map_shapes"]:
        n = 3 * int(h) * int(w)
        out.append(z["maps"][at:at + n].reshape(3, int(h), int(w)))
        at += n
    return out


def render_args(rec, sizes):
    """The arguments of render_init_maps / render_fixed / render_serial for a Reconstruction and its image sizes."""
    from esac_b200.prepare import camera_geometry
    geo = [camera_geometry(rec.kind, h, w) for h, w in sizes]
    return (rec.points, rec.offsets, rec.indices, rec.poses, rec.focal, np.array([g[2] for g in geo]),
            [(g[0], g[1]) for g in geo])
