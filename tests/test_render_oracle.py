"""The init-map renderer's restatements (oracle/render_oracle.py) and esac_b200.prepare's readers and writer, held to the
reference's converters on the fixtures of tests/golden/render/ (written by make_render_golden.py from the reference's own
create_training_set / create_set).  No GPU: the writer is fed render_fixed's maps."""
from pathlib import Path

import numpy as np
import pytest
import torch

from esac_b200 import prepare
from oracle.render_oracle import (fixed_product, fixture_maps, fixture_reconstruction, render_args, render_fixed,
                                  render_serial)

FIXTURES = sorted((Path(__file__).resolve().parent / "golden" / "render").glob("*.npz"))
IDS = [p.stem for p in FIXTURES]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_bits(xs, ys):
    return len(xs) == len(ys) and all(x.shape == y.shape and np.array_equal(bits(x), bits(y)) for x, y in zip(xs, ys))


def saved(z, rec, maps):
    """The maps of the cameras the reference saved, in its order."""
    by_name = {n[:-4]: m for n, m in zip(rec.names, maps)}
    return [by_name[str(n)] for n in z["saved"]]


def test_fixtures_cover_both_kinds():
    assert IDS == ["aachen_generic", "dubrovnik_exact", "dubrovnik_generic"]


@pytest.mark.parametrize("npz", FIXTURES, ids=IDS)
def test_readers_reproduce_camera_and_observation_order(npz, tmp_path):
    z, rec, _ = fixture_reconstruction(npz, tmp_path)
    counts = z["cam_counts"]
    assert len(rec.names) == len(counts)
    assert np.array_equal(np.diff(rec.offsets), counts)
    assert np.array_equal(bits(rec.points[rec.indices]), bits(z["cam_points"]))
    names = [n[:-4] for n in rec.names]
    assert [str(n) for n in z["saved"]] == [n for n in names if n in set(str(s) for s in z["saved"])]


@pytest.mark.parametrize("npz", FIXTURES, ids=IDS)
def test_serial_loop_with_torch_mm_reproduces_the_reference(npz, tmp_path):
    z, rec, sizes = fixture_reconstruction(npz, tmp_path)
    maps, _, _ = render_serial(*render_args(rec, sizes), product="torch")
    assert same_bits(saved(z, rec, maps), fixture_maps(z))


@pytest.mark.parametrize("npz", FIXTURES, ids=IDS)
def test_fixed_order_reproduces_the_reference(npz, tmp_path):
    z, rec, sizes = fixture_reconstruction(npz, tmp_path)
    maps, zbufs, counts, status = render_fixed(*render_args(rec, sizes))
    assert not status.any()
    assert same_bits(saved(z, rec, maps), fixture_maps(z))


@pytest.mark.parametrize("npz", FIXTURES, ids=IDS)
def test_writer_reproduces_the_reference_files(npz, tmp_path):
    z, rec, sizes = fixture_reconstruction(npz, tmp_path)
    maps, zbufs, _, _ = render_fixed(*render_args(rec, sizes))
    empty = [rec.kind == "dubrovnik" and not (zb != 0).any() for zb in zbufs]
    written, skipped = prepare.save_training_files(str(tmp_path / "out"), rec, sizes, maps, empty)
    assert [n[:-4] for n in written] == [str(n) for n in z["saved"]]
    assert len(written) + len(skipped) == len(rec.names)
    for k, n in enumerate(z["saved"]):
        n = str(n)
        m = torch.load(tmp_path / "out" / "init" / (n + ".dat"))
        assert m.dtype == torch.float32 and m.untyped_storage().nbytes() == m.numel() * 4
        assert np.array_equal(bits(m.numpy()), bits(fixture_maps(z)[k]))
        assert (tmp_path / "out" / "calibration" / (n + ".txt")).read_text() == str(z["calib"][k])
        pose = np.array([float(v) for v in (tmp_path / "out" / "poses" / (n + ".txt")).read_text().split()]).reshape(4, 4)
        np.testing.assert_allclose(pose, z["poses"][k], rtol=1e-6, atol=1e-6)


def test_exact_fixture_holds_the_edge_cases(tmp_path):
    """What the exact scene is there for: a tie, a negative depth winning, depth-0 points written and not written, and a
    camera skipped for an empty z-buffer."""
    npz = next(p for p in FIXTURES if p.stem == "dubrovnik_exact")
    z, rec, sizes = fixture_reconstruction(npz, tmp_path)
    maps, zbufs, counts, _ = render_fixed(*render_args(rec, sizes))
    m0, z0 = maps[0], zbufs[0]
    assert list(m0[:, 30, 40]) == [0.0625, 0.0625, 4]        # equal depths: the earlier point
    assert list(m0[:, 34, 44]) == [-0.5, -0.5, -4]           # a negative depth beats the nearer positive ones
    assert list(m0[:, 59, 79]) == [50, 50, 6]                # a farther point after a depth 0
    assert list(m0[:, 0, 0]) == [-5, -5, 0] and z0[0, 0] == 0  # a depth 0 alone: written, z-buffer 0
    assert list(m0[:, 59, 0]) == [-9, 9, 0]                  # the last of two depth-0 points
    assert list(m0[:, 0, 79]) == [-20, 30, -1]               # a depth 0 after a negative depth is not written
    assert list(maps[1][:, 0, 59]) == [3, 5, -2]             # a depth 0 after a positive depth is written
    assert (zbufs[2] <= 0).all() and (zbufs[2] < 0).any()    # only points behind the camera
    assert counts[-1] == 0 and [n[:-4] for n in rec.names][-1] not in set(str(s) for s in z["saved"])


def adversarial(seed, C=6):
    """Small-integer points and axis-aligned integer poses: ties, depth-0 points, negative depths, clamps and duplicate
    observations are frequent, and every pose product is exact.  Observations whose projection is NaN are dropped."""
    rng = np.random.default_rng(seed)
    shapes = [(int(rng.integers(1, 6)), int(rng.integers(1, 6))) for _ in range(C)]
    pts = rng.integers(-3, 4, (40, 3)).astype(np.float32)
    poses = np.zeros((C, 3, 4), np.float32)
    for c in range(C):
        perm, sign = rng.permutation(3), rng.choice([-1, 1], 3)
        poses[c, np.arange(3), perm] = sign
        poses[c, :, 3] = rng.integers(-2, 3, 3)
    cam = np.repeat(np.arange(C), rng.integers(0, 30, C))
    idx = rng.integers(0, len(pts), len(cam))
    cp = fixed_product(poses[cam], pts[idx])
    keep = ~((cp[:, 2] == 0) & ((cp[:, 0] == 0) | (cp[:, 1] == 0)))
    cam, idx = cam[keep], idx[keep].astype(np.int32)
    offsets = np.concatenate([[0], np.cumsum(np.bincount(cam, minlength=C))])
    return pts, offsets, idx, poses, rng.choice([0.5, 1.0, 2.0], C), rng.choice([0.5, 1.0], C), shapes


@pytest.mark.parametrize("seed", range(40))
def test_fixed_order_equals_the_serial_loop_on_adversarial_inputs(seed):
    args = adversarial(seed)
    ms, zs, cs = render_serial(*args, product="fixed")
    mf, zf, cf, st = render_fixed(*args)
    assert not st.any()
    assert same_bits(ms, mf) and same_bits(zs, zf) and np.array_equal(cs, cf)
    mt, zt, ct = render_serial(*args, product="torch")  # exact products: torch.mm agrees too
    assert same_bits(mt, mf) and same_bits(zt, zf) and np.array_equal(ct, cf)


def test_nan_projection_is_flagged_and_the_loop_raises():
    pts = np.array([[0, 1, 0], [1, 1, 1]], np.float32)   # the first: cam = (0, 1, 0) under the identity
    args = (pts, np.array([0, 1, 2]), np.array([1, 0], np.int32), np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)),
            [1.0, 1.0], [1.0, 1.0], [(4, 4), (4, 4)])
    _, _, _, status = render_fixed(*args)
    assert list(status) == [0, 2]
    with pytest.raises(ValueError):
        render_serial(*args)
    bad = (pts, np.array([0, 1]), np.array([2], np.int32), np.eye(4, dtype=np.float32)[None], [1.0], [1.0], [(4, 4)])
    assert list(render_fixed(*bad)[3]) == [1]


def test_camera_geometry_of_both_kinds():
    # Aachen: 480 px short side, then ceil(/8), with the calibration factor img_w / width; Dubrovnik: 60 cells straight away
    assert prepare.camera_geometry("aachen", 45, 80)[:2] == (60, 107)
    assert prepare.camera_geometry("dubrovnik", 45, 80)[:2] == (60, 107)
    assert prepare.camera_geometry("aachen", 683, 1024)[:2] == (60, 90)
    assert prepare.camera_geometry("aachen", 1024, 683) == (90, 60, 60 / 683, 480 / 683)
    assert prepare.camera_geometry("dubrovnik", 1024, 683) == (90, 60, 60 / 683, 1.0)
    assert prepare.camera_geometry("aachen", 480, 640) == (60, 80, 0.125, 1.0)
