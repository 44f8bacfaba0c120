"""GPU tests of the hypotheses node's probability floor (minProb / min_prob, run with `-m gpu`): the explicit default is the
default bit for bit in all three forms; at floor 0 every hypothesis is refined as the oracle refines it and each term of
the gradient meets the float64 oracle at that floor (tests/floor_terms.py) on its own scale; an intermediate floor flags
exactly p >= floor; batched, ragged and stream-ordered calls are the single eager call row by row; a captured graph
replays the eager floor-0 node; E = 20, M = 1024 at 480x640 completes; and the best-of-M example checks itself."""
import contextlib
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import floor_terms as FT
import grad_terms as GT
from esac_b200.synth import make_scene, pose_error
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
TAIL = (10.0, 100.0, 0.5, 100.0)    # tau, alpha, beta, maxReproj
# E = 2, 30x40, M = 32: 26 hypotheses below PROB_THRESH, down to p ~ 1e-21
FLOOR_SCENE, FLOOR_SEED = dict(E=2, H=30, W=40, M=32, sub=8, seed=1), 71
BAR_NODE = 1e-6   # tests/test_gpu_backward_terms.py's bar for the node against the oracle fed the same upstream


@contextlib.contextmanager
def _own_context():
    """A context of its own on device 0 (fixed_seed off), so that its stream-ordered workspace has seen only this code."""
    import esac_b200.api as api
    saved = api._contexts.get(0)
    ctx = api.Context(0)
    api._contexts[0] = ctx
    try:
        yield api
    finally:
        import torch
        torch.cuda.synchronize()
        if saved is not None:
            api._contexts[0] = saved
        else:
            api._contexts.pop(0, None)
        ctx.close()


@pytest.fixture(scope="module")
def api():
    with _own_context() as api:
        yield api


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _upstream(M, k):
    rng = np.random.default_rng(900 + k)
    return rng.standard_normal(M), rng.standard_normal((M, 6))


def _eager(api, sc, seed, up, **floor):
    """hypotheses_forward then hypotheses_backward with upstream `up` (scores, poses): numpy outputs and gradient.  seed
    None: the next call of the context's sequence."""
    import torch
    coords = _cuda(sc.coords)
    if seed is not None:
        api.set_seed(seed)
    scores, poses, contrib, tape = api.hypotheses_forward(coords, _cuda(sc.assign), *sc.params, **floor)
    st = api.last_stats()
    probs = api.last_hypotheses()["probs"].copy()
    g = torch.zeros_like(coords)
    api.hypotheses_backward(tape, coords, g, _cuda(up[0]), _cuda(up[1]))
    return dict(scores=_np(scores), poses=_np(poses), contrib=_np(contrib), grad=_np(g), n_contrib=st["n_contrib"],
                probs=probs)


def _same(a, b, keys=("scores", "poses", "contrib", "grad")):
    """Bitwise equal outputs (a one-image batch against its single call)."""
    for k in keys:
        np.testing.assert_array_equal(np.reshape(a[k], np.shape(b[k])), b[k], err_msg=k)


def test_explicit_default_floor_is_the_default_bitwise(api):
    """minProb=1e-3 passed explicitly: outputs, and tapes through their gradients, bitwise the default call's."""
    import torch
    sc = make_scene(**FLOOR_SCENE)
    up = _upstream(sc.assign.shape[0], 0)
    a, b = _eager(api, sc, 5, up), _eager(api, sc, 5, up, minProb=1e-3)
    _same(a, b)
    assert a["n_contrib"] == b["n_contrib"] == int((a["probs"] >= O.PROB_THRESH).sum()) >= 2
    # batch
    scenes = [make_scene(**{**FLOOR_SCENE, "seed": 10 + k}) for k in range(3)]
    coords = _cuda(np.stack([s.coords for s in scenes]))
    assign = _cuda(np.stack([s.assign for s in scenes]))
    outs = []
    for floor in ({}, {"minProb": 1e-3}):
        api.set_seed(6)
        s_, p_, c_, tapes = api.hypotheses_forward_batch(coords, assign, *scenes[0].params, **floor)
        g = torch.zeros_like(coords)
        api.hypotheses_backward_batch(tapes, coords, g, _cuda(np.stack([up[0]] * 3)), _cuda(np.stack([up[1]] * 3)))
        outs.append(dict(scores=_np(s_), poses=_np(p_), contrib=_np(c_), grad=_np(g)))
    _same(*outs)
    # stream-ordered
    outs = [_async_node(api, [sc], [up], 7, floor) for floor in ({}, {"minProb": 1e-3})]
    _same(*outs)


def _async_node(api, scenes, ups, seed, floor):
    """hypotheses_forward_async + hypotheses_backward_async of B images of one shape, uncaptured."""
    import torch
    B = len(scenes)
    E, _, H, W = scenes[0].coords.shape
    M, sub = scenes[0].assign.shape[0], scenes[0].sub
    coords = _cuda(np.stack([s.coords for s in scenes]))
    tapes = torch.zeros(B * api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, device="cuda")
    z = dict(device="cuda")
    scores, poses = torch.zeros(B, M, dtype=torch.float64, **z), torch.zeros(B, M, 6, dtype=torch.float64, **z)
    contrib, st = torch.zeros(B, M, dtype=torch.bool, **z), torch.full((B,), 7, dtype=torch.int32, **z)
    shifts = torch.tensor([[s.shiftX, s.shiftY] for s in scenes], dtype=torch.int32, **z)
    cams = torch.tensor([[s.f, s.ppx, s.ppy] for s in scenes], dtype=torch.float32, **z)
    api.set_seed(seed)
    api.hypotheses_forward_async(coords, _cuda(np.stack([s.assign for s in scenes])), shifts, cams, *TAIL, sub, tapes, scores,
                                 poses, contrib, st, **floor)
    g = torch.zeros_like(coords)
    bst = api.hypotheses_backward_async(tapes, coords, g, M, _cuda(np.stack([u[0] for u in ups])),
                                        _cuda(np.stack([u[1] for u in ups])))
    assert (st.cpu() == 0).all() and (bst.cpu() == 0).all()
    return dict(scores=_np(scores), poses=_np(poses), contrib=_np(contrib), grad=_np(g))


@pytest.fixture(scope="module")
def floor_zero(api):
    """The floor scene's forward at minProb=0 on the GPU (fixed_seed on): (scene, CUDA coordinates, tape, outputs)."""
    sc = make_scene(**FLOOR_SCENE)
    coords = _cuda(sc.coords)
    api.context().set_option("fixed_seed", 1)
    try:
        api.set_seed(FLOOR_SEED)
        scores, poses, contrib, tape = api.hypotheses_forward(coords, _cuda(sc.assign), *sc.params, minProb=0.0)
        probs = api.last_hypotheses()["probs"].copy()
        n = api.last_stats()["n_contrib"]
    finally:
        api.context().set_option("fixed_seed", 0)
    return sc, coords, tape, dict(scores=_np(scores), poses=_np(poses), contrib=_np(contrib), probs=probs, n_contrib=n)


def test_floor_zero_refines_every_hypothesis_as_the_oracle(floor_zero):
    sc, _, _, out = floor_zero
    M = sc.assign.shape[0]
    assert out["contrib"].all() and out["n_contrib"] == M
    _, tr = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, FLOOR_SEED, None, None, prob_thresh=0.0)
    assert np.abs(out["scores"] - np.array(tr.scores)).max() < 1e-4
    below = np.nonzero(tr.probs < O.PROB_THRESH)[0]
    assert len(below) >= 16 and (out["probs"][below] < O.PROB_THRESH).all()
    moved = 0
    for h in range(M):
        mine = O.pose2trans(out["poses"][h, :3], out["poses"][h, 3:]).astype(np.float32)
        want = O.pose2trans(*tr.ref[h]).astype(np.float32)
        rot, trans = pose_error(mine, want)
        assert rot < 1e-3 and trans < 1e-5, (h, tr.probs[h], rot, trans)
        init = np.r_[tr.hyps[h].rvec.ravel(), tr.hyps[h].tvec.ravel()]
        moved += h in below and not np.array_equal(out["poses"][h], init)
    assert moved >= 8   # hypotheses below PROB_THRESH now leave the node refined


def _node_against_floor_oracle(api, floor_zero, gp, gs, what):
    import torch
    sc, coords, tape, _ = floor_zero
    g = torch.zeros(sc.coords.shape, device="cuda")
    api.hypotheses_backward(tape, coords, g, None if gs is None else _cuda(gs), None if gp is None else _cuda(gp))
    g_ref, tr = FT.hypotheses_vjp(sc.coords, sc.assign, *sc.params, FLOOR_SEED, gp, gs, prob_thresh=0.0)
    assert np.abs(g_ref).max() > 0
    rep = GT.assert_classwise(_np(g), g_ref, FT.cell_classes(sc.coords.shape, sc.assign, tr), BAR_NODE, what)
    print(f"{what}: {GT.fmt(rep)}")
    return rep, tr


def _best_of_m_upstream(sc, out):
    """d/d(scores, poses) of min_h reference_pose_loss(pose_h) + 1e-3 * mean_h (that loss) - 0.01 * mean(scores): non-zero
    on every hypothesis's pose and score."""
    M = sc.assign.shape[0]
    gt = sc.gt_pose.astype(np.float64)
    gt_r, gt_t = O.trans2pose(gt)
    losses = np.array([O.loss(O.pose2trans(q[:3], q[3:]), gt, 1.0, 100.0, 100.0) for q in out["poses"]])
    dl = np.array([O.d_loss(q[:3], q[3:], gt_r, gt_t, 1.0, 100.0, 100.0).ravel() for q in out["poses"]])
    w = np.full(M, 1e-3 / M)
    w[int(np.argmin(losses))] += 1.0
    return w[:, None] * dl, np.full(M, -0.01 / M)


def test_floor_zero_direct_term_meets_the_oracle(api, floor_zero):
    _, gs = _best_of_m_upstream(floor_zero[0], floor_zero[3])
    _node_against_floor_oracle(api, floor_zero, None, np.linspace(-1.0, 1.0, gs.size), "path II")


def test_floor_zero_path_one_meets_the_oracle(api, floor_zero):
    gp, _ = _best_of_m_upstream(floor_zero[0], floor_zero[3])
    assert (np.abs(gp).max(1) > 0).all()
    rep, tr = _node_against_floor_oracle(api, floor_zero, gp, None, "path I")
    assert rep["inlier"]["scale"] > 0


def test_floor_zero_best_of_m_loss_meets_the_oracle(api, floor_zero):
    gp, gs = _best_of_m_upstream(floor_zero[0], floor_zero[3])
    rep, tr = _node_against_floor_oracle(api, floor_zero, gp, gs, "best-of-M")
    assert rep["minimal"]["cells"] > 0 and rep["rest"]["cells"] > 0


def test_intermediate_floor_flags_exactly_p_at_or_above_it(api):
    sc = make_scene(**FLOOR_SCENE)
    up = _upstream(sc.assign.shape[0], 1)
    for floor in (1e-6, 1e-12):
        r = _eager(api, sc, 9, up, minProb=floor)
        assert np.array_equal(r["contrib"], r["probs"] >= floor)
        assert r["n_contrib"] == int(r["contrib"].sum())
        assert int((r["probs"] >= O.PROB_THRESH).sum()) < r["n_contrib"] < sc.assign.shape[0] or floor == 1e-12


def test_batched_and_ragged_rows_are_single_calls(api):
    import torch
    scenes = [make_scene(**{**FLOOR_SCENE, "seed": 20 + k, "shiftX": k, "f": 500.0 + 20 * k}) for k in range(3)]
    M = scenes[0].assign.shape[0]
    ups = [_upstream(M, 10 + k) for k in range(3)]
    for ragged in (False, True):
        if ragged:  # maps of different sizes
            crops = [(30, 40), (27, 35), (24, 40)]
            scenes = [make_scene(**{**FLOOR_SCENE, "H": h, "W": w, "seed": 20 + k, "shiftX": k, "f": 500.0 + 20 * k})
                      for k, (h, w) in enumerate(crops)]
            coords = [_cuda(s.coords) for s in scenes]
        else:
            coords = _cuda(np.stack([s.coords for s in scenes]))
        assign = _cuda(np.stack([s.assign for s in scenes]))
        cams = tuple([getattr(s, k) for s in scenes] for k in ("shiftX", "shiftY", "f", "ppx", "ppy"))
        # image b of the batch draws what the b-th of B consecutive single calls after set_seed draws
        api.set_seed(33)
        want = [_eager(api, sc, None, up, minProb=0.0) for sc, up in zip(scenes, ups)]
        api.set_seed(33)
        s_, p_, c_, tapes = api.hypotheses_forward_batch(coords, assign, *cams, *TAIL, 8, minProb=0.0)
        g = [torch.zeros_like(c) for c in coords] if ragged else torch.zeros_like(coords)
        api.hypotheses_backward_batch(tapes, coords, g, _cuda(np.stack([u[0] for u in ups])),
                                      _cuda(np.stack([u[1] for u in ups])))
        for b, w in enumerate(want):
            assert w["contrib"].all()
            row = dict(scores=_np(s_[b]), poses=_np(p_[b]), contrib=_np(c_[b]), grad=_np(g[b]))
            _same(row, w)


def test_stream_ordered_floor_zero_is_the_eager_node_and_replays_from_a_graph(api):
    import torch
    scenes = [make_scene(**{**FLOOR_SCENE, "seed": 40 + k}) for k in range(3)]
    E, _, H, W = scenes[0].coords.shape
    M, sub = scenes[0].assign.shape[0], scenes[0].sub
    ups = [_upstream(M, 20 + k) for k in range(3)]
    eager = [_eager(api, sc, 44 + k, up, minProb=0.0) for k, (sc, up) in enumerate(zip(scenes, ups))]
    # uncaptured: each image the first call after set_seed(44 + k), as its eager twin
    refs = []
    for k, (sc, up) in enumerate(zip(scenes, ups)):
        refs.append(_async_node(api, [sc], [up], 44 + k, {"minProb": 0.0}))
    for r, e in zip(refs, eager):
        assert e["contrib"].all()
        _same(r, e)
    # captured with minProb = 0, replayed with new inputs and seeds
    api.reserve_backward_async(1, E, H, W, M, sub)
    z = dict(device="cuda")
    coords, assign = torch.zeros(1, E, 3, H, W, **z), torch.zeros(1, M, dtype=torch.int64, **z)
    shifts, cams = torch.zeros(1, 2, dtype=torch.int32, **z), torch.ones(1, 3, **z)
    tapes = torch.zeros(api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, **z)
    scores, poses = torch.zeros(1, M, dtype=torch.float64, **z), torch.zeros(1, M, 6, dtype=torch.float64, **z)
    contrib, fst, bst = (torch.zeros(1, M, dtype=torch.bool, **z), torch.full((1,), 7, dtype=torch.int32, **z),
                         torch.full((1,), 7, dtype=torch.int32, **z))
    d_s, d_p, grads = torch.zeros(1, M, dtype=torch.float64, **z), torch.zeros(1, M, 6, dtype=torch.float64, **z), \
        torch.zeros(1, E, 3, H, W, **z)

    def write(sc, up):
        coords[0].copy_(_cuda(sc.coords)); assign[0].copy_(_cuda(sc.assign)); grads.zero_()
        shifts[0].copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
        cams[0].copy_(torch.tensor([sc.f, sc.ppx, sc.ppy]))
        d_s[0].copy_(_cuda(up[0])); d_p[0].copy_(_cuda(up[1]))

    def step():
        api.hypotheses_forward_async(coords, assign, shifts, cams, *TAIL, sub, tapes, scores, poses, contrib, fst, minProb=0.0)
        api.hypotheses_backward_async(tapes, coords, grads, M, d_s, d_p, bst)

    write(scenes[0], ups[0])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for k, (sc, up, e) in enumerate(zip(scenes, ups, eager)):
        write(sc, up)
        api.set_seed(44 + k)
        graph.replay()
        assert int(fst[0]) == 0 and int(bst[0]) == 0
        _same(dict(scores=_np(scores[0]), poses=_np(poses[0]), contrib=_np(contrib[0]), grad=_np(grads[0])), e)


def test_floor_zero_at_e20_m1024_full_size_completes():
    """Every one of 1 024 hypotheses refined and differentiated at 480x640 (sub 1) with 20 experts, eager and
    stream-ordered: status 0, everything contributes, finite outputs.  A fresh context: the module's stream-ordered
    workspace is frozen by the capture above."""
    with _own_context() as api:
        _full_size(api)


def _full_size(api):
    import torch
    E, H, W, M = 20, 480, 640, 1024
    sc = make_scene(E=E, H=H, W=W, M=M, sub=1, seed=5, per_expert=False)
    coords = _cuda(sc.coords)
    api.set_seed(3)
    scores, poses, contrib, tape = api.hypotheses_forward(coords, _cuda(sc.assign), *sc.params, minProb=0.0)
    assert bool(contrib.all()) and api.last_stats()["n_contrib"] == M
    assert bool(torch.isfinite(scores).all()) and bool(torch.isfinite(poses).all())
    g = torch.zeros_like(coords)
    up = _upstream(M, 3)
    api.hypotheses_backward(tape, coords, g, _cuda(up[0]), _cuda(up[1]))
    assert bool(torch.isfinite(g).all()) and float(g.abs().max()) > 0
    del tape
    api.reserve_backward_async(1, E, H, W, M, 1)
    out = _async_node(api, [sc], [up], 3, {"minProb": 0.0})
    assert out["contrib"].all() and np.isfinite(out["grad"]).all()
    _same(out, dict(scores=_np(scores), poses=_np(poses), contrib=_np(contrib), grad=_np(g)))


def test_best_of_m_example_checks_against_the_eager_step():
    r = subprocess.run([sys.executable, str(ROOT / "examples" / "best_of_m_step_synthetic.py"), "--steps", "3", "--check"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "bitwise" in r.stdout
