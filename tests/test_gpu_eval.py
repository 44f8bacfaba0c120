"""The pose evaluation on the device (esac_b200/csrc/eval.cu, api.evaluate_poses[_async], esac_b200.evaluate.PoseEvaluator)
against the float64 oracle (oracle/eval_oracle.py), batch against single calls, captured against eager, the store's
overflow, and the reference's test loop end to end (examples/test_eval_graph_synthetic.py)."""
import functools
import importlib.util
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.evaluate import PoseEvaluator
from oracle import eval_oracle as O
from orientations import cam_to_world, rotate, uniform_rotations

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=1)
def _pairs():
    """10k (estimate, ground truth) pairs: uniform rotations at room and world scale, and the edge sets of
    tests/test_eval_oracle.py (angles straddling s = 1e-5, identity, 179 to 180 degrees, slightly non-orthonormal)."""
    rng = np.random.default_rng(11)
    rots = uniform_rotations(12000, seed=17)
    P, G = [], []
    for i in range(0, 12000, 2):
        scale = 1000.0 if i % 8 == 0 else 3.0
        c = rng.uniform(-1, 1, 3) * scale
        P.append(cam_to_world(rots[i], c))
        G.append(cam_to_world(rots[i + 1], c + rng.uniform(-2, 2, 3)))
    for k, R in enumerate(uniform_rotations(500, seed=23)):
        axis = rng.normal(size=3)
        for ang in (0.8e-5, 1.2e-5, math.radians(179.0), math.radians(179.5), math.radians(179.9), math.pi, 0.0):
            P.append(cam_to_world(rotate(R, axis, ang)))
            G.append(cam_to_world(R))
        if k < 50:   # an estimate whose rotation is the identity: the pose file's q_xyz is NaN
            P.append(cam_to_world(np.eye(3), rng.uniform(-3, 3, 3)))
            G.append(cam_to_world(R))
        skew = cam_to_world(rots[k])
        skew[:3, :3] += rng.uniform(-3e-4, 3e-4, (3, 3)).astype(np.float32)
        P.append(skew)
        G.append(cam_to_world(rots[k + 1]))
    return np.stack(P), np.stack(G)


def _inputs(B, E=5, seed=0):
    rng = np.random.default_rng(seed)
    experts = torch.from_numpy(rng.integers(0, E, B)).cuda()
    scenes = torch.from_numpy(rng.integers(0, E, B)).cuda()
    hist = torch.from_numpy((rng.random((B, E)) < 0.4).astype(np.float32) * rng.integers(1, 9, (B, E)).astype(np.float32)).cuda()
    status = torch.from_numpy(rng.integers(0, 3, B).astype(np.int32)).cuda()
    return experts, scenes, hist, status


def test_records_equal_the_oracle():
    P, G = _pairs()
    B = len(P)
    experts, scenes, hist, status = _inputs(B)
    rec = api.evaluate_poses(torch.from_numpy(P).cuda(), torch.from_numpy(G).cuda(), experts, scenes, hist=hist,
                             status=status).cpu().numpy()
    ref = O.evaluate_batch(P, G, experts.cpu().numpy(), scenes.cpu().numpy(), hist.cpu().numpy(), status.cpu().numpy())
    assert rec.shape == (B, 14) and B >= 10000
    # flags, scene, expert, status and experts active exactly
    assert np.array_equal(rec[:, 2:7], ref[:, 2:7])
    # rotation within 1e-9 deg, wider where acos is ill-conditioned: c may differ by dc = 2e-15 (fp64 rounding through the
    # Newton steps, contracted differently on the device), so theta by dc / sin(theta), at most sqrt(2 dc) (next to 180 deg)
    theta = np.radians(ref[:, 0])
    cond = np.degrees(np.minimum(2e-15 / np.maximum(np.sin(theta), 1e-300), math.sqrt(4e-15)))
    assert np.all(np.abs(rec[:, 0] - ref[:, 0]) <= 1e-9 + cond), np.abs(rec[:, 0] - ref[:, 0]).max()
    assert np.array_equal(rec[:, 0] == 0, ref[:, 0] == 0)
    assert np.all(np.abs(rec[:, 1] - ref[:, 1]) <= 1e-9 * np.maximum(ref[:, 1], 1e-3))
    # t within 1e-12 (of the translation's scale), q within 1e-12 up to its sign (at 180 degrees the axis' sign is a
    # rounding decision), NaN where the oracle's is
    tscale = 1 + np.linalg.norm(ref[:, 11:14], axis=1)
    assert np.all(np.abs(rec[:, 11:14] - ref[:, 11:14]).max(axis=1) <= 1e-12 * tscale)
    nan = np.isnan(ref[:, 8:11]).any(axis=1)
    assert np.array_equal(nan, np.isnan(rec[:, 8:11]).any(axis=1)) and nan.sum() >= 50
    dq = np.minimum(np.abs(rec[~nan, 7:11] - ref[~nan, 7:11]).max(axis=1), np.abs(rec[~nan, 7:11] + ref[~nan, 7:11]).max(axis=1))
    assert dq.max() <= 1e-12, dq.max()


def test_single_pose_and_no_histogram():
    P, G = _pairs()
    rec = api.evaluate_poses(torch.from_numpy(P[0]).cuda(), torch.from_numpy(G[0]).cuda(),
                             torch.tensor(3).cuda(), torch.tensor(3).cuda()).cpu().numpy()
    ref = O.evaluate(P[0], G[0], 3, 3)
    assert rec.shape == (14,) and rec[2] == 1.0 and rec[5] == 0.0 and math.isnan(rec[6]) and math.isnan(ref[6])
    assert abs(rec[0] - ref[0]) <= 1e-9 and np.allclose(rec[7:], ref[7:], rtol=0, atol=1e-12)


def _bits(t):
    return t.contiguous().view(torch.int64)


def test_batch_equals_single_calls_and_slots_are_consecutive():
    """B = 300 images: three CTAs read the counter of one launch."""
    P, G = _pairs()
    B = 300
    Pd, Gd = torch.from_numpy(P[:B]).cuda(), torch.from_numpy(G[:B]).cuda()
    experts, scenes, hist, status = _inputs(B, seed=4)
    batch, single = PoseEvaluator(5, 2 * B), PoseEvaluator(5, 2 * B)
    batch.update(Pd[:7], Gd[:7], experts[:7], scenes[:7], hist=hist[:7], status=status[:7])
    batch.update(Pd[7:], Gd[7:], experts[7:], scenes[7:], hist=hist[7:], status=status[7:])
    for b in range(B):
        single.update(Pd[b], Gd[b], experts[b], scenes[b], hist=hist[b], status=status[b])
    assert int(batch.state[0]) == int(single.state[0]) == B and int(batch.state[2]) == 0
    assert torch.equal(_bits(batch.buffer[:B]), _bits(single.buffer[:B]))
    whole = api.evaluate_poses(Pd, Gd, experts, scenes, hist=hist, status=status)
    assert torch.equal(_bits(whole), _bits(batch.buffer[:B]))


def test_captured_update_equals_eager_updates():
    K, B = 6, 9
    P, G = _pairs()
    Pd, Gd = torch.from_numpy(P[:B]).cuda(), torch.from_numpy(G[:B]).cuda()
    experts, scenes, hist, status = _inputs(B, seed=5)
    eager, captured = PoseEvaluator(5, K * B), PoseEvaluator(5, K * B)
    for _ in range(K):
        eager.update(Pd, Gd, experts, scenes, hist=hist, status=status)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        captured.update(Pd, Gd, experts, scenes, hist=hist, status=status)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured.update(Pd, Gd, experts, scenes, hist=hist, status=status)
    captured.reset()
    for _ in range(K):
        graph.replay()
    assert torch.equal(_bits(torch.from_numpy(captured.records())), _bits(torch.from_numpy(eager.records())))
    assert captured.records().shape == (K * B, 14)


def test_overflow_keeps_the_first_records_and_records_raises():
    K = 5
    P, G = _pairs()
    Pd, Gd = torch.from_numpy(P[:K + 3]).cuda(), torch.from_numpy(G[:K + 3]).cuda()
    experts, scenes, hist, status = _inputs(K + 3, seed=6)
    ev = PoseEvaluator(5, K)
    for b in range(K + 3):
        ev.update(Pd[b], Gd[b], experts[b], scenes[b], hist=hist[b], status=status[b])
    state = ev.state.cpu().tolist()
    assert state[:3] == [K + 3, 1, 0]
    whole = api.evaluate_poses(Pd[:K], Gd[:K], experts[:K], scenes[:K], hist=hist[:K], status=status[:K])
    assert torch.equal(_bits(ev.buffer), _bits(whole))
    with pytest.raises(RuntimeError, match=f"capacity {K}"):
        ev.records()
    ev.reset()
    assert ev.records().shape == (0, 14)


def _example(name):
    sys.path.insert(0, str(ROOT / "examples"))
    spec = importlib.util.spec_from_file_location(name, ROOT / "examples" / f"{name}.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture
def own_context():
    """The example runs on a context of its own, whose stream-ordered workspace no earlier capture has frozen; cuDNN's
    flags are restored after."""
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    saved = api._contexts.get(0)
    api._contexts[0] = api.Context(0)
    yield
    torch.cuda.synchronize()
    if saved is not None:
        api._contexts[0] = saved
    else:
        api._contexts.pop(0, None)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


def _off_boundary(x, decimals, margin):
    """x is more than `margin` from every rounding boundary of `decimals` decimals."""
    scaled = x * 10 ** decimals
    return abs(scaled - math.floor(scaled) - 0.5) > margin * 10 ** decimals


def test_example_loop_gives_the_host_evaluation(own_context, capsys, tmp_path):
    """The gated test step with the evaluator in the graph over SyntheticRoomDataset images: the same table, results file
    and pose file as the oracle on the read-back poses.  No compared value may lie within 1e-6 of a threshold or of a
    console rounding boundary (two decimals for the medians); the results file prints six
    decimals, whose boundaries lie 1e-6 apart, so there the margin is 1e-12."""
    mod = _example("test_eval_graph_synthetic")
    opt = mod.options(["--images", "24", "--experts", "6", "--check", "--outdir", str(tmp_path)])
    r = mod.run(opt)
    assert r["table"]["console"] == r["host_table"]["console"]
    assert r["table"]["results"] == r["host_table"]["results"]
    assert r["table"]["experts"] == r["host_table"]["experts"]
    assert r["pose_lines"] == r["host_pose_lines"]
    rec, host = r["records"], r["host_records"]
    assert np.array_equal(rec[:, 2:7], host[:, 2:7])
    counted = rec[:, 5] == 0
    assert counted.sum() >= 12
    for v in np.concatenate([rec[counted, 0], rec[counted, 1]]):
        assert abs(v - 5.0) > 1e-6
    for row in r["table"]["rows"]:
        for v in row[3:]:   # the medians (the accuracies are ratios of counts, the same arithmetic on both sides)
            assert _off_boundary(v, 2, 1e-6) and _off_boundary(v, 6, 1e-12), row
    rc = mod.main(["--images", "24", "--experts", "6", "--check", "--outdir", str(tmp_path)])
    out = capsys.readouterr().out
    assert rc == 0 and "same table and pose file" in out, out
    assert (tmp_path / "results_esac_synthetic.txt").read_text().splitlines() == r["table"]["results"]
    assert (tmp_path / "poses_esac_synthetic.txt").read_text().splitlines() == r["pose_lines"]
