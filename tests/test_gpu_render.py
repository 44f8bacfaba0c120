"""The init-map renderer (esac_b200/csrc/render.cu, api.render_init_maps) held bitwise to oracle/render_oracle.py's
render_fixed: coordinate planes, z-buffers, written-cell counts and status, on the golden fixtures (whose maps are the
reference's) and on edge cases, small and large."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import prepare
from esac_b200.cluster import cluster_environment
from esac_b200.synth import make_reconstruction
from oracle.render_oracle import fixture_maps, fixture_reconstruction, render_args, render_fixed

pytestmark = pytest.mark.gpu
FIXTURES = sorted((Path(__file__).resolve().parent / "golden" / "render").glob("*.npz"))


def bits(a):
    if torch.is_tensor(a):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check(args, cuda_inputs=False):
    """Kernel == render_fixed bitwise; returns the kernel's maps and counts."""
    points, offsets, indices, poses, focal, scale, shapes = args
    want_m, want_z, want_c, want_s = render_fixed(*args)
    assert not want_s.any()
    if cuda_inputs:
        points = torch.as_tensor(np.asarray(points, np.float32)).cuda()
        indices = torch.as_tensor(np.asarray(indices, np.int32)).cuda()
    maps, counts, zbufs = api.render_init_maps(points, offsets, indices, poses, focal, scale, shapes, zbuffer=True)
    assert len(maps) == len(want_m) and all(m.is_cuda for m in maps)
    for c in range(len(maps)):
        assert tuple(maps[c].shape) == want_m[c].shape
        assert np.array_equal(bits(maps[c]), bits(want_m[c])), f"camera {c}: maps differ"
        assert np.array_equal(bits(zbufs[c]), bits(want_z[c])), f"camera {c}: z-buffers differ"
    assert np.array_equal(counts.numpy(), want_c)
    return maps, counts


@pytest.mark.parametrize("npz", FIXTURES, ids=[p.stem for p in FIXTURES])
@pytest.mark.parametrize("cuda_inputs", [False, True], ids=["host", "cuda"])
def test_golden_fixtures(npz, cuda_inputs, tmp_path):
    z, rec, sizes = fixture_reconstruction(npz, tmp_path)
    args = render_args(rec, sizes)
    maps, _ = check(args, cuda_inputs)
    by_name = {n[:-4]: m for n, m in zip(rec.names, maps)}
    for n, ref in zip(z["saved"], fixture_maps(z)):
        assert np.array_equal(bits(by_name[str(n)]), bits(ref))   # the reference's own maps


def test_write_training_set_matches_the_reference_files(tmp_path):
    npz = next(p for p in FIXTURES if p.stem == "dubrovnik_exact")
    z, rec, sizes = fixture_reconstruction(npz, tmp_path)
    out = prepare.write_training_set(str(tmp_path / "out"), rec, sizes)
    assert [n[:-4] for n in out.names] == [str(n) for n in z["saved"]]
    assert out.skipped == [rec.names[-1]]
    for k, n in enumerate(z["saved"]):
        m = torch.load(tmp_path / "out" / "init" / (str(n) + ".dat"))
        assert not m.is_cuda and m.untyped_storage().nbytes() == m.numel() * 4
        assert np.array_equal(bits(m), bits(fixture_maps(z)[k]))
        assert (tmp_path / "out" / "calibration" / (str(n) + ".txt")).read_text() == str(z["calib"][k])


def one_camera(pts, idx, shape=(6, 8), pose=None, f=4.0, s=1.0):
    pose = np.eye(4, dtype=np.float32) if pose is None else pose
    return (np.asarray(pts, np.float32).reshape(-1, 3), np.array([0, len(idx)]), np.asarray(idx, np.int32), pose[None],
            [f], [s], [shape])


def test_one_camera():
    rng = np.random.default_rng(1)
    pts = np.concatenate([rng.uniform(-1, 1, (300, 2)), rng.uniform(1, 5, (300, 1))], 1)
    check(one_camera(pts, rng.integers(0, 300, 900)))


def test_camera_without_observations_and_zero_observations():
    pts = np.array([[0.1, 0.2, 2.0]], np.float32)
    args = (pts, np.array([0, 0, 2, 2]), np.array([0, 0], np.int32), np.tile(np.eye(4, dtype=np.float32), (3, 1, 1)),
            [4.0] * 3, [1.0] * 3, [(6, 8), (5, 5), (3, 7)])
    maps, counts = check(args)
    assert counts.tolist() == [0, 1, 0] and not maps[0].any() and not maps[2].any()
    maps, counts = check((pts, np.array([0, 0]), np.zeros(0, np.int32), np.eye(4, dtype=np.float32)[None], [4.0], [1.0],
                          [(4, 4)]))   # V = 0
    assert counts.tolist() == [0] and not maps[0].any()
    maps, counts = check((np.zeros((0, 3), np.float32), np.array([0, 0]), np.zeros(0, np.int32),
                          np.eye(4, dtype=np.float32)[None], [4.0], [1.0], [(1, 1)]))   # P = 0 too
    assert counts.tolist() == [0]


def test_only_points_behind_the_camera():
    rng = np.random.default_rng(2)
    pts = np.concatenate([rng.uniform(-3, 3, (200, 2)), rng.uniform(-5, -0.5, (200, 1))], 1)
    maps, counts = check(one_camera(pts, np.arange(200)))
    assert counts.item() > 0


def test_exact_scene_and_repeat_bitwise(tmp_path):
    npz = next(p for p in FIXTURES if p.stem == "dubrovnik_exact")
    _, rec, sizes = fixture_reconstruction(npz, tmp_path)
    args = render_args(rec, sizes)
    m1, c1 = check(args)
    m2, c2 = check(args, cuda_inputs=True)
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(m1, m2)) and torch.equal(c1, c2)


def test_large_reconstruction_and_repeat_bitwise():
    r = make_reconstruction(seed=7, cameras=4000, points=1_000_000)
    rec = r["rec"]
    assert rec.offsets[-1] >= 5_000_000
    args = (rec.points, rec.offsets, rec.indices, rec.poses, rec.focal, r["out_scale"], r["shapes"])
    m1, c1 = check(args, cuda_inputs=True)
    m2, c2, _ = api.render_init_maps(*args)
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(m1, m2)) and torch.equal(c1, c2)


def test_bad_index_and_nan_projection_raise_naming_the_camera():
    pts = np.array([[0, 1, 0], [1, 1, 1]], np.float32)   # the first projects to NaN under the identity
    eye = np.tile(np.eye(4, dtype=np.float32), (3, 1, 1))
    with pytest.raises(RuntimeError, match=r"2 camera\(s\) cannot be rendered: 0 \(a point index out of range\), "
                                           r"2 \(a NaN projection\)"):
        api.render_init_maps(pts, np.array([0, 2, 3, 4]), np.array([1, 5, 1, 0], np.int32), eye, [4.0] * 3, [1.0] * 3,
                             [(4, 4)] * 3)
    with pytest.raises(RuntimeError, match=r"0 \(a point index out of range\)"):
        api.render_init_maps(torch.as_tensor(pts).cuda(), np.array([0, 1]), torch.tensor([-1], dtype=torch.int32).cuda(),
                             eye[:1], 4.0, 1.0, [(4, 4)])
    torch.cuda.synchronize()
    check(one_camera(pts[1:], [0]))   # the context still works


def test_c_entry_refuses_inconsistent_arguments(lib):
    ctx = api.context()
    h = ctx.handle
    out = torch.zeros(3 * 16, device="cuda")
    cnt, st = np.zeros(2, np.int32), np.zeros(2, np.int32)
    pts = torch.zeros(2, 3, device="cuda")
    idx = torch.zeros(2, dtype=torch.int32, device="cuda")
    poses = np.tile(np.eye(4, dtype=np.float32)[:3], (2, 1, 1))
    f = np.ones(2, np.float32)
    H = np.array([2, 2], np.int32)
    W = np.array([4, 4], np.int32)

    def call(C_=2, offs=(0, 1, 2), P=2, Hs=H, Ws=W, maps=out.data_ptr(), count=cnt.ctypes.data, indices=idx.data_ptr(),
             points=pts.data_ptr()):
        o = np.asarray(offs, np.int64)
        return lib.esacb200_render_init_maps(h, C_, points, P, o.ctypes.data, indices, poses.ctypes.data,
                                             f.ctypes.data, f.ctypes.data, Hs.ctypes.data, Ws.ctypes.data, maps, None,
                                             count, st.ctypes.data)

    assert call() == 0
    for kwargs, msg in [(dict(C_=0), "0 cameras"), (dict(offs=(1, 1, 2)), "offsets[0]=1"), (dict(offs=(0, 2, 1)),
                        "offsets decrease at camera 1"), (dict(P=-1), "P=-1"), (dict(Hs=np.array([2, 0], np.int32)),
                        "camera 1 map is 0x4"), (dict(Ws=np.array([8193, 4], np.int32)), "camera 0 map is 2x8193"),
                        (dict(maps=None), "null pointer"), (dict(count=None), "null pointer"),
                        (dict(indices=None), "2 observations but indices is null"),
                        (dict(points=None), "2 points but points is null"),
                        (dict(maps=cnt.ctypes.data), "out_maps is host memory")]:
        assert call(**kwargs) == -2, kwargs
        assert msg in lib.esacb200_last_error(h).decode(), (kwargs, lib.esacb200_last_error(h))
    assert call() == 0
    assert call(P=0, points=None) == 0 and list(st) == [1, 1]   # no points: every index is out of range, flagged


def test_no_points_raises_naming_the_cameras():
    with pytest.raises(RuntimeError, match=r"2 camera\(s\) cannot be rendered: 0 \(a point index out of range\), 1 \("):
        api.render_init_maps(np.zeros((0, 3), np.float32), np.array([0, 1, 3]), np.array([0, 0, 2], np.int32),
                             np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)), 4.0, 1.0, [(4, 4), (3, 5)])


def test_host_inputs_are_ordered_after_pending_torch_work():
    """The outputs come from torch's caching allocator: a block freed while torch work on it is still queued can come back
    at once.  The render must run on torch's current stream so that the queued write lands before it, not after."""
    rng = np.random.default_rng(4)
    pts = np.concatenate([rng.uniform(-1, 1, (5000, 2)), rng.uniform(1, 5, (5000, 1))], 1)
    args = one_camera(pts, rng.integers(0, 5000, 20000), shape=(120, 160), f=100.0)
    want = render_fixed(*args)[0][0]
    torch.cuda.synchronize()
    stale = torch.empty(3 * 120 * 160, device="cuda")
    ptr = stale.data_ptr()
    torch.cuda._sleep(200_000_000)   # keeps the fill below queued for a while (about 0.1 s)
    stale.fill_(7.0)
    del stale
    maps, _, _ = api.render_init_maps(*args)
    assert maps[0].data_ptr() == ptr   # the allocator handed the same block back
    torch.cuda.synchronize()
    assert np.array_equal(bits(maps[0]), bits(want))


def test_clustering_the_rendered_maps_matches_the_oracle_maps():
    r = make_reconstruction(seed=3, cameras=300, points=60_000)
    rec = r["rec"]
    args = (rec.points, rec.offsets, rec.indices, rec.poses, rec.focal, r["out_scale"], r["shapes"])
    maps, _, _ = api.render_init_maps(*args)
    want = render_fixed(*args)[0]
    a = cluster_environment(maps, num_clusters=8, seed=5)
    b = cluster_environment([torch.as_tensor(m).cuda() for m in want], num_clusters=8, seed=5)
    assert torch.equal(a.labels, b.labels)
