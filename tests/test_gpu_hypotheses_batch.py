"""The batched hypotheses node (autograd.esac_hypotheses_batch, api.hypotheses_forward_batch / hypotheses_backward_batch,
batched api.pose_loss) on the GPU: bitwise equality with loops of the single-image node, the reference loss against
backward_batch, stacked against list, input kinds and streams, the batched pose loss against the oracle, tapes, graph and
memory, errors that name the image, and the batched custom-loss example (run with `-m gpu`)."""
import numpy as np
import pytest

from esac_b200.synth import make_scene
from oracle import esac_oracle as O

pytestmark = pytest.mark.gpu

# portrait and landscape, N = H * W = 1200, 1107 (odd), 775 (odd), 1408
SHAPES = [(30, 40), (41, 27), (25, 31), (44, 32)]
W_LOSS = (1.0, 100.0, 100.0)


def _scenes(shapes=SHAPES, E=3, M=48, seed=70):
    """A batch with its own focal length, principal point and shift per image."""
    return [make_scene(E=E, H=h, W=w, M=M, sub=8, seed=seed + b, outlier_frac=0.6, f=480.0 + 15 * b, ppx=4 * w + 3 * b - 4,
                       ppy=4 * h - 2 * b + 1, shiftX=b - 1, shiftY=2 - b) for b, (h, w) in enumerate(shapes)]


def _batch(scenes, device="cuda"):
    """(maps list, assignment [B,M], ground truths [B,4,4], the ten per-batch parameters with per-image cameras)."""
    import torch
    coords = [torch.from_numpy(s.coords).to(device) for s in scenes]
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).to(device)
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).to(device)
    cams = [[getattr(s, k) for s in scenes] for k in ("shiftX", "shiftY", "f", "ppx", "ppy")]
    return coords, assign, gts, cams + list(scenes[0].params[5:])


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    ctx = api.context()
    ctx.set_option("fixed_seed", 0)
    ctx.set_option("batch_workers", 8)
    yield api
    ctx.set_option("batch_workers", 8)


def _np(*ts):
    return [t.detach().cpu().numpy() for t in ts]


def test_forward_equals_a_loop_of_single_calls(api):
    scenes = _scenes()
    coords, assign, _, params = _batch(scenes)
    B = len(scenes)
    api.set_seed(31)
    s, p, c, tapes = api.hypotheses_forward_batch(coords, assign, *params)
    nxt = api.hypotheses_forward(coords[0], assign[0], *scenes[0].params)
    api.set_seed(31)
    loop = [api.hypotheses_forward(coords[b], assign[b], *scenes[b].params) for b in range(B)]
    after = api.hypotheses_forward(coords[0], assign[0], *scenes[0].params)
    assert len(tapes) == B and all(t.data_ptr() % 256 == 0 for t in tapes)
    assert len({t.untyped_storage().data_ptr() for t in tapes}) == 1
    for b in range(B):
        for x, y in zip(_np(s[b], p[b], c[b]), _np(*loop[b][:3])):
            assert np.array_equal(x, y), b
        assert c[b].any()
    for x, y in zip(_np(*nxt[:3]), _np(*after[:3])):
        assert np.array_equal(x, y)


@pytest.fixture(scope="module")
def fwd(api):
    scenes = _scenes()
    coords, assign, _, params = _batch(scenes)
    api.set_seed(33)
    s, p, c, tapes = api.hypotheses_forward_batch(coords, assign, *params)
    return scenes, coords, tapes, c


@pytest.mark.parametrize("workers", [1, 8])
@pytest.mark.parametrize("up", ["both", "scores", "poses", "none"])
def test_backward_equals_a_loop_of_single_calls(api, fwd, workers, up):
    import torch
    scenes, coords, tapes, contrib = fwd
    B, M = contrib.shape
    rng = np.random.default_rng(5)
    gs = torch.tensor(rng.normal(size=(B, M)), device="cuda") if up in ("both", "scores") else None
    gp = torch.tensor(rng.normal(size=(B, M, 6)) * 1e-2, device="cuda") if up in ("both", "poses") else None
    start = [torch.from_numpy(rng.normal(size=c.shape).astype(np.float32)).cuda() for c in coords]
    grads = [g.clone() for g in start]
    api.context().set_option("batch_workers", workers)
    try:
        api.hypotheses_backward_batch(tapes, coords, grads, gs, gp)
    finally:
        api.context().set_option("batch_workers", 8)
    for b in range(B):
        g = start[b].clone()
        api.hypotheses_backward(tapes[b], coords[b], g, None if gs is None else gs[b], None if gp is None else gp[b])
        assert torch.equal(grads[b], g), b
        assert torch.equal(g, start[b]) == (up == "none"), b


@pytest.mark.parametrize("kind", ["stacked", "list"])
def test_reference_loss_through_the_batched_node_is_backward_batch(api, kind):
    import torch
    from esac_b200.autograd import esac_hypotheses_batch, reference_pose_loss
    scenes = _scenes() if kind == "list" else _scenes([(30, 40)] * 4)
    coords, assign, gts, params = _batch(scenes)
    B = len(scenes)
    x = [c.clone().requires_grad_(True) for c in coords] if kind == "list" else torch.stack(coords).requires_grad_(True)
    api.set_seed(41)
    scores, poses, contrib = esac_hypotheses_batch(x, assign, *params)
    losses = (torch.softmax(scores, 1) * reference_pose_loss(poses, gts, *W_LOSS)).sum(1)
    losses.sum().backward()
    g = [t.grad for t in x] if kind == "list" else list(x.grad)
    api.set_seed(41)
    g_ref = [torch.zeros_like(c) for c in coords] if kind == "list" else torch.zeros_like(x)
    l_ref = api.backward_batch(coords if kind == "list" else torch.stack(coords), g_ref, assign, gts, *W_LOSS, *params)
    api.set_seed(41)
    n_contrib = []
    for b in range(B):  # a batch call keeps only the last image's statistics
        api.backward(coords[b], torch.zeros_like(coords[b]), assign[b], gts[b], *W_LOSS, *scenes[b].params)
        n_contrib.append(api.last_stats()["n_contrib"])
    assert contrib.sum(1).tolist() == n_contrib and min(n_contrib) >= 1
    for b in range(B):
        assert abs(losses[b].item() - l_ref[b]) <= 1e-12 * abs(l_ref[b]), (b, losses[b].item(), l_ref[b])
        scale = g_ref[b].abs().max().item()
        assert scale > 0
        assert (g[b] - g_ref[b]).abs().max().item() <= 1e-6 * scale, b


def _run(api, x, assign, params, seed, a, b_):
    """Outputs and coordinate gradients of the batched node for fixed upstreams a [B,M,6], b_ [B,M] (numpy)."""
    import torch
    from esac_b200.autograd import esac_hypotheses_batch
    x = [t.detach().requires_grad_(True) for t in x] if isinstance(x, list) else x.detach().requires_grad_(True)
    api.set_seed(seed)
    scores, poses, contrib = esac_hypotheses_batch(x, assign, *params)
    g = torch.autograd.grad((scores, poses), x, (torch.tensor(b_, device=scores.device), torch.tensor(a, device=poses.device)))
    return _np(scores, poses, contrib) + _np(*g)


def test_a_list_of_equal_shapes_is_bitwise_the_stacked_call(api):
    import torch
    scenes = _scenes([(30, 40)] * 4)
    coords, assign, _, params = _batch(scenes)
    rng = np.random.default_rng(6)
    a, b_ = rng.normal(size=(4, 48, 6)) * 1e-2, rng.normal(size=(4, 48))
    stacked = _run(api, torch.stack(coords), assign, params, 43, a, b_)
    listed = _run(api, coords, assign, params, 43, a, b_)
    assert np.abs(stacked[3]).max() > 0
    for x, y in zip(stacked[:3], listed[:3]):
        assert np.array_equal(x, y)
    assert np.array_equal(stacked[3], np.stack(listed[3:]))


def test_cpu_cuda_and_misaligned_inputs_give_the_same_bits_and_calls_follow_the_stream(api):
    import torch
    scenes = _scenes()
    coords, assign, _, params = _batch(scenes)
    rng = np.random.default_rng(7)
    a, b_ = rng.normal(size=(4, 48, 6)) * 1e-2, rng.normal(size=(4, 48))
    misaligned = []
    for c in coords:
        buf = torch.zeros(c.numel() + 1, device="cuda")
        m = buf[1:].view(c.shape)
        m.copy_(c)
        assert m.data_ptr() % 16 == 4
        misaligned.append(m)
    runs = [_run(api, [c.cpu() for c in coords], assign.cpu(), params, 47, a, b_), _run(api, coords, assign, params, 47, a, b_),
            _run(api, misaligned, assign, params, 47, a, b_)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        # the maps are produced on the side stream right before the call: the node must run after them
        late = []
        for c in coords:
            slow = torch.zeros(c.shape, device="cuda")
            for _ in range(50):
                slow = slow * 1.0001
            late.append(slow * 0 + c)
        runs.append(_run(api, late, assign, params, 47, a, b_))
    s.synchronize()
    assert np.abs(runs[0][3]).max() > 0
    for r in runs[1:]:
        for x, y in zip(r, runs[0]):
            assert np.array_equal(x, y)


def test_batched_pose_loss_is_per_image_and_meets_the_oracle(api):
    import torch
    from esac_b200.autograd import reference_pose_loss
    scenes = _scenes()
    B, M = len(scenes), 40
    rng = np.random.default_rng(3)
    rows = []
    for s in scenes:  # 2 to 60 degrees and 1 cm to 3 m away from each image's ground truth
        gt_r, gt_t = O.trans2pose(s.gt_pose.astype(np.float64))
        img = []
        for _ in range(M):
            ax = rng.normal(size=3)
            dr = ax / np.linalg.norm(ax) * np.radians(rng.uniform(2, 60))
            img.append(np.r_[gt_r.ravel() + dr, gt_t.ravel() + rng.normal(size=3) * 10 ** rng.uniform(-2, 0.5)])
        rows.append(img)
    rows = np.array(rows)
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    poses = torch.tensor(rows, dtype=torch.float64, device="cuda", requires_grad=True)
    for w_rot, w_trans in ((1.0, 100.0), (1.0, 0.0)):
        l_all = np.array([[O.loss(O.pose2trans(p[:3], p[3:]), s.gt_pose.astype(np.float64), w_rot, w_trans, 1e9) for p in img]
                          for s, img in zip(scenes, rows)])
        cut = float(np.float32(np.median(l_all)))
        losses, dloss = api.pose_loss(poses.detach(), gts, w_rot, w_trans, cut)
        for b in range(B):
            lb, db = api.pose_loss(poses.detach()[b], gts[b], w_rot, w_trans, cut)
            assert torch.equal(losses[b], lb) and torch.equal(dloss[b], db), b
        up = torch.linspace(0.5, 2.0, B * M, dtype=torch.float64, device="cuda").view(B, M)
        lo = reference_pose_loss(poses, gts, w_rot, w_trans, cut)
        assert torch.equal(lo.detach(), losses)
        g, = torch.autograd.grad((lo * up).sum(), poses)
        g = (g / up[..., None]).cpu().numpy()
        lo = lo.detach().cpu().numpy()
        above = 0
        for b, s in enumerate(scenes):
            gt64 = s.gt_pose.astype(np.float64)
            gt_r, gt_t = O.trans2pose(gt64)
            for i, p in enumerate(rows[b]):
                lr = O.loss(O.pose2trans(p[:3], p[3:]), gt64, w_rot, w_trans, cut)
                above += lr > cut
                dl = O.d_loss(p[:3], p[3:], gt_r, gt_t, w_rot, w_trans, cut).ravel()
                assert abs(lo[b, i] - lr) <= 1e-11 * max(1.0, abs(lr)), (b, i, lo[b, i], lr)
                assert np.abs(g[b, i] - dl).max() <= 1e-9 * max(1.0, np.abs(dl).max()), (b, i, g[b, i], dl)
        assert 0 < above < B * M


def test_tapes_are_independent_of_later_calls(api):
    import torch
    batches = [_scenes(), _scenes([(24, 33), (36, 28)], E=2, M=32, seed=90)]
    rng = np.random.default_rng(12)
    ups = [(rng.normal(size=(len(s), s[0].assign.shape[0], 6)) * 1e-2, rng.normal(size=(len(s), s[0].assign.shape[0])))
           for s in batches]
    data = [_batch(s) for s in batches]

    def fwd(i):
        coords, assign, _, params = data[i]
        api.set_seed(60 + i)
        return api.hypotheses_forward_batch(coords, assign, *params)

    def bwd(i, tapes):
        coords = data[i][0]
        g = [torch.zeros_like(c) for c in coords]
        api.hypotheses_backward_batch(tapes, coords, g, torch.tensor(ups[i][1], device="cuda"),
                                      torch.tensor(ups[i][0], device="cuda"))
        return _np(*g)

    alone = []
    for i in range(2):
        out = fwd(i)
        alone.append((_np(*out[:3]), bwd(i, out[3])))
    out0, out1 = fwd(0), fwd(1)
    g1, g0 = bwd(1, out1[3]), bwd(0, out0[3])     # backwards in reverse order, after both forwards
    for i, (out, g) in enumerate(((out0, g0), (out1, g1))):
        for x, y in zip(_np(*out[:3]), alone[i][0]):
            assert np.array_equal(x, y)
        for x, y in zip(g, alone[i][1]):
            assert np.array_equal(x, y)
        assert max(np.abs(x).max() for x in g) > 0


def test_retain_graph_and_memory(api):
    import torch
    from esac_b200.autograd import esac_hypotheses_batch, pose_to_transform
    scenes = _scenes()
    coords0, assign, gts, params = _batch(scenes)

    def step():
        coords = [c.clone().requires_grad_(True) for c in coords0]
        api.set_seed(57)
        scores, poses, contrib = esac_hypotheses_batch(coords, assign, *params)
        T = pose_to_transform(poses)
        L = (torch.softmax(scores, 1) * (T[..., :3, 3] - gts[:, None, :3, 3].double()).norm(dim=-1)).sum()
        g1 = torch.autograd.grad(L, coords, retain_graph=True)
        g2 = torch.autograd.grad(L, coords)
        for a, b in zip(g1, g2):
            assert torch.equal(a, b) and a.abs().max() > 0

    step()  # first use of the batched matmul allocates torch's persistent library workspaces
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    step()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == base


def test_an_expert_index_out_of_range_names_the_image(api):
    scenes = _scenes()
    coords, assign, _, params = _batch(scenes)
    bad = assign.clone()
    bad[2, 5] = 3  # E = 3
    with pytest.raises(RuntimeError, match=r"image 2: hypAssignment holds an expert index outside \[0, 3\)"):
        api.hypotheses_forward_batch(coords, bad, *params)
    api.set_seed(31)
    s, *_ = api.hypotheses_forward_batch(coords, assign, *params)   # the workers are usable afterwards
    assert s.isfinite().all()


def test_batched_custom_loss_example_checks_against_esac_loss_batch():
    import runpy
    import sys
    from pathlib import Path
    ex = Path(__file__).resolve().parents[1] / "examples" / "custom_loss_batch_step_synthetic.py"
    argv = sys.argv
    sys.argv = [str(ex), "--steps", "3", "--check"]
    try:
        mod = runpy.run_path(str(ex), run_name="example")
        assert mod["main"]() == 0
    finally:
        sys.argv = argv
