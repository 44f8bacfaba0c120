"""GPU tests of the stream-ordered hypotheses node (api.hypotheses_forward_async / hypotheses_backward_async /
pose_loss_async and autograd.esac_hypotheses_async): bitwise equal to the eager node call for call, graph replays with new
inputs, seeds and cameras, batches, one call counter with backward_async, no host synchronisation, the per-image status,
the workspace rule, independent tapes, captured training steps, and the graph example (run with `-m gpu`)."""
import numpy as np
import pytest

from esac_b200.synth import make_scene

pytestmark = pytest.mark.gpu

LOSS = (1.0, 100.0, 100.0)          # wLossRot, wLossTrans, lossCut
TAIL = (10.0, 100.0, 0.5, 100.0)    # tau, alpha, beta, maxReproj

SHAPES = [  # E, H, W, M, sub: the shapes of test_gpu_backward_async.py
    (1, 60, 80, 64, 8),
    (7, 60, 80, 256, 8),
    (7, 480, 640, 256, 1),
    (2, 40, 27, 64, 8),
    (3, 61, 107, 96, 8),
]


@pytest.fixture(scope="module")
def api():
    """The module's own context, so that the stream-ordered workspace here has seen only these tests."""
    import esac_b200.api as api
    saved = api._contexts.get(0)
    ctx = api.Context(0)
    api._contexts[0] = ctx
    ctx.set_option("fixed_seed", 0)
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


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _scenes(n, E, H, W, M, sub, seed, **kw):
    """n images whose shift, focal length and principal point all differ."""
    return [make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=seed + k, f=480.0 + 37.5 * k, ppx=W * sub / 2 + 3.25 * k - 4,
                       ppy=H * sub / 2 - 2.5 * k + 1, shiftX=k - 2, shiftY=1 - k, **kw) for k in range(n)]


def _varied_scenes(E, H, W, M, sub):
    """From clean to mostly outliers: the refinement group the eager node picks differs between them."""
    return [make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=300 + k, f=500.0 + 40.0 * k, ppx=W * sub / 2 + k, ppy=H * sub / 2 - k,
                       shiftX=2 - k, shiftY=k - 3, outlier_frac=frac, noise=noise)
            for k, (frac, noise) in enumerate([(0.4, 0.02), (0.9, 0.3), (0.1, 0.005), (0.8, 0.15), (0.95, 0.5), (0.6, 0.05)])]


def _upstream(sc, k):
    """A random upstream and a non-zero starting gradient (the backward accumulates)."""
    rng = np.random.default_rng(2000 + k)
    M = sc.assign.shape[0]
    return (rng.standard_normal(M), rng.standard_normal((M, 6)),
            (rng.standard_normal(sc.coords.shape) * 1e-3).astype(np.float32))


def _eager(api, sc, up):
    """The eager node: hypotheses_forward then hypotheses_backward on device tensors.  Returns (scores, poses, contrib,
    gradient, refinement group)."""
    coords = _cuda(sc.coords)
    scores, poses, contrib, tape = api.hypotheses_forward(coords, _cuda(sc.assign), *sc.params)
    group = api.last_stats()["refine_group"]
    grads = _cuda(up[2].copy())
    api.hypotheses_backward(tape, coords, grads, _cuda(up[0]), _cuda(up[1]))
    return scores.cpu().numpy(), poses.cpu().numpy(), contrib.cpu().numpy(), grads.cpu().numpy(), group


class Node:
    """The static inputs and outputs of B images of one shape through the stream-ordered node."""

    def __init__(self, api, B, E, H, W, M, sub):
        import torch
        self.api, self.B, self.M, self.sub = api, B, M, sub
        z = dict(device="cuda")
        self.coords = torch.zeros(B, E, 3, H, W, **z)
        self.grads = torch.zeros(B, E, 3, H, W, **z)
        self.assign = torch.zeros(B, M, dtype=torch.int64, **z)
        self.shifts = torch.zeros(B, 2, dtype=torch.int32, **z)
        self.cameras = torch.ones(B, 3, **z)
        self.d_scores = torch.zeros(B, M, dtype=torch.float64, **z)
        self.d_poses = torch.zeros(B, M, 6, dtype=torch.float64, **z)
        self.tapes = torch.zeros(B * api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, **z)
        self.scores = torch.zeros(B, M, dtype=torch.float64, **z)
        self.poses = torch.zeros(B, M, 6, dtype=torch.float64, **z)
        self.contrib = torch.zeros(B, M, dtype=torch.bool, **z)
        self.fstatus = torch.full((B,), 7, dtype=torch.int32, **z)
        self.bstatus = torch.full((B,), 7, dtype=torch.int32, **z)

    def write(self, scenes, ups):
        import torch
        for b, (sc, up) in enumerate(zip(scenes, ups)):
            self.coords[b].copy_(_cuda(sc.coords))
            self.assign[b].copy_(_cuda(sc.assign))
            self.shifts[b].copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
            self.cameras[b].copy_(torch.tensor([sc.f, sc.ppx, sc.ppy], dtype=torch.float32))
            self.d_scores[b].copy_(_cuda(up[0]))
            self.d_poses[b].copy_(_cuda(up[1]))
            self.grads[b].copy_(_cuda(up[2]))

    def forward(self):
        self.api.hypotheses_forward_async(self.coords, self.assign, self.shifts, self.cameras, *TAIL, self.sub, self.tapes,
                                          self.scores, self.poses, self.contrib, self.fstatus)

    def backward(self):
        self.api.hypotheses_backward_async(self.tapes, self.coords, self.grads, self.M, self.d_scores, self.d_poses,
                                           self.bstatus)

    def both(self):
        self.forward()
        self.backward()

    def results(self, b=0):
        return (self.scores[b].cpu().numpy(), self.poses[b].cpu().numpy(), self.contrib[b].cpu().numpy(),
                self.grads[b].cpu().numpy())

    def assert_eager(self, ref, b=0):
        assert int(self.fstatus[b]) == 0 and int(self.bstatus[b]) == 0, (self.fstatus, self.bstatus)
        for mine, want in zip(self.results(b), ref[:4]):
            np.testing.assert_array_equal(mine, want)


def _capture(fn):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "E%d_%dx%d_M%d_sub%d" % s)
def test_calls_one_to_five_equal_eager_node_bitwise(api, shape):
    import torch
    E, H, W, M, sub = shape
    scenes = _scenes(5, E, H, W, M, sub, seed=100 + E + H)
    ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
    api.set_seed(4242)
    ref = [_eager(api, sc, up) for sc, up in zip(scenes, ups)]
    assert any(r[2].any() for r in ref)
    api.set_seed(4242)
    node = Node(api, 1, E, H, W, M, sub)
    for sc, up, r in zip(scenes, ups, ref):
        node.write([sc], [up])
        node.both()
        node.assert_eager(r)
    # one image may also be passed unbatched
    api.set_seed(4242)
    sc, up = scenes[0], ups[0]
    z = dict(device="cuda")
    scores, poses = torch.zeros(M, dtype=torch.float64, **z), torch.zeros(M, 6, dtype=torch.float64, **z)
    contrib, status = torch.zeros(M, dtype=torch.bool, **z), torch.zeros((), dtype=torch.int32, **z)
    tape = torch.zeros(api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, **z)
    coords, grads = _cuda(sc.coords), _cuda(up[2].copy())
    api.hypotheses_forward_async(coords, _cuda(sc.assign), torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, **z),
                                 torch.tensor([sc.f, sc.ppx, sc.ppy], **z), *TAIL, sub, tape, scores, poses, contrib, status)
    bst = api.hypotheses_backward_async(tape, coords, grads, M, _cuda(up[0]), _cuda(up[1]))
    assert int(status) == 0 and int(bst) == 0
    for mine, want in zip((scores, poses, contrib, grads), ref[0][:4]):
        np.testing.assert_array_equal(mine.cpu().numpy(), want)


def _replay_and_compare(g, node, scenes, ups, ref, between=None):
    for r, (sc, up, rf) in enumerate(zip(scenes, ups, ref)):
        node.write([sc], [up])
        if between:
            between(r)
        g.replay()
        node.assert_eager(rf)


def test_graph_replays_with_new_inputs_seeds_and_cameras(api):
    E, H, W, M, sub = 3, 60, 80, 256, 8
    scenes = _varied_scenes(E, H, W, M, sub)
    ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
    api.reserve_backward_async(1, E, H, W, M, sub)
    node = Node(api, 1, E, H, W, M, sub)
    node.write([scenes[0]], [ups[0]])
    g = _capture(node.both)
    api.set_seed(77)
    ref = [_eager(api, sc, up) for sc, up in zip(scenes, ups)]
    groups = [r[4] for r in ref]
    assert len(set(groups)) >= 2, groups   # the device picks the group per replay
    api.set_seed(77)
    _replay_and_compare(g, node, scenes, ups, ref)
    # set_seed between replays takes effect at the next replay
    api.set_seed(78)
    ref = [_eager(api, sc, up) for sc, up in zip(scenes[:2], ups[:2])]
    api.set_seed(91)
    ref += [_eager(api, sc, up) for sc, up in zip(scenes[2:], ups[2:])]
    api.set_seed(78)
    _replay_and_compare(g, node, scenes, ups, ref, between=lambda r: api.set_seed(91) if r == 2 else None)
    # fixed_seed, as captured
    ctx = api.context()
    ctx.set_option("fixed_seed", 1)
    try:
        g_fixed = _capture(node.both)
        api.set_seed(123)
        ref = [_eager(api, sc, up) for sc, up in zip(scenes[:3], ups[:3])]
        api.set_seed(123)
        _replay_and_compare(g_fixed, node, scenes[:3], ups[:3], ref)
    finally:
        ctx.set_option("fixed_seed", 0)


def test_batch_equals_hypotheses_batch_row_by_row(api):
    import torch
    E, H, W, M, sub = 3, 30, 40, 48, 8
    scenes = _scenes(4, E, H, W, M, sub, seed=500)
    ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
    coords = _cuda(np.stack([s.coords for s in scenes]))
    cams = ([s.shiftX for s in scenes], [s.shiftY for s in scenes], [s.f for s in scenes], [s.ppx for s in scenes],
            [s.ppy for s in scenes])
    api.set_seed(555)
    scores, poses, contrib, tapes = api.hypotheses_forward_batch(coords, _cuda(np.stack([s.assign for s in scenes])), *cams,
                                                                 *TAIL, sub)
    grads = _cuda(np.stack([u[2] for u in ups]))
    api.hypotheses_backward_batch(tapes, coords, grads, _cuda(np.stack([u[0] for u in ups])), _cuda(np.stack([u[1] for u in ups])))
    node = Node(api, 4, E, H, W, M, sub)
    node.write(scenes, ups)
    api.set_seed(555)
    node.both()
    assert (node.fstatus.cpu() == 0).all() and (node.bstatus.cpu() == 0).all()
    assert torch.equal(node.scores, scores) and torch.equal(node.poses, poses) and torch.equal(node.contrib, contrib)
    assert torch.equal(node.grads, grads)


def test_backward_async_and_node_share_the_call_counter(api):
    import torch
    E, H, W, M, sub = 3, 60, 80, 64, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=450)
    ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
    api.reserve_backward_async(1, E, H, W, M, sub)
    node = Node(api, 1, E, H, W, M, sub)
    bgrads = torch.zeros_like(node.grads)
    gt = torch.eye(4, device="cuda")[None].clone()
    loss, lstatus = torch.zeros(1, dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")

    def both():
        api.backward_async(node.coords, bgrads, node.assign, gt, node.shifts, node.cameras, *LOSS, *TAIL, sub, loss, lstatus)
        node.both()

    g = _capture(both)
    api.set_seed(5150)
    ref = []
    for sc, up in zip(scenes, ups):   # eager: esac.backward (call 2r), then the node (call 2r + 1)
        eg = torch.zeros(1, E, 3, H, W, device="cuda")
        lo = api.backward(_cuda(sc.coords), eg[0], _cuda(sc.assign), _cuda(sc.gt_pose), *LOSS, *sc.params)
        ref.append(((lo, eg.cpu().numpy()), _eager(api, sc, up)))
    api.set_seed(5150)
    for sc, up, (bref, nref) in zip(scenes, ups, ref):
        node.write([sc], [up])
        gt[0].copy_(_cuda(sc.gt_pose))
        bgrads.zero_()
        g.replay()
        assert int(lstatus[0]) == 0 and float(loss[0]) == bref[0]
        np.testing.assert_array_equal(bgrads.cpu().numpy(), bref[1])
        node.assert_eager(nref)


def test_no_host_synchronisation(api):
    import torch
    E, H, W, M, sub = 2, 60, 80, 64, 8
    sc = _scenes(1, E, H, W, M, sub, seed=600)[0]
    up = _upstream(sc, 0)
    api.reserve_backward_async(1, E, H, W, M, sub)
    node = Node(api, 1, E, H, W, M, sub)
    node.write([sc], [up])
    gt = _cuda(sc.gt_pose)[None]
    out_l = torch.zeros(1, M, dtype=torch.float64, device="cuda")
    out_d = torch.zeros(1, M, 6, dtype=torch.float64, device="cuda")
    calls = {"forward": node.forward, "backward": node.backward,
             "pose_loss_async": lambda: api.pose_loss_async(node.poses, gt, *LOSS, out_l, out_d)}
    node.both()
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    for name, fn in calls.items():
        torch.cuda._sleep(int(2e9))       # ~1 s of device time ahead of the call
        fn()
        assert not stream.query(), f"{name} waited for the device"
        torch.cuda.synchronize()
    # captured in torch's default (global) error mode, with torch work before and after, and replayed
    src = node.coords.clone()
    doubled = torch.zeros_like(out_l)
    for name, fn in calls.items():
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            node.coords.copy_(src * 1.0)
            fn()
            doubled.copy_(out_l * 2.0)
        torch.cuda.synchronize()
        torch.cuda._sleep(int(2e9))
        g.replay()
        assert not stream.query(), f"the replay of {name} waited for the device"
        torch.cuda.synchronize()
    assert int(node.fstatus[0]) == 0 and int(node.bstatus[0]) == 0
    np.testing.assert_array_equal(doubled.cpu().numpy(), 2.0 * out_l.cpu().numpy())


def test_status_of_a_bad_expert_index_and_of_a_foreign_tape(api):
    import torch
    E, H, W, M, sub = 3, 30, 40, 48, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=700)
    ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
    scenes[1].assign[5] = E   # outside [0, E)
    api.set_seed(999)
    ref0 = _eager(api, scenes[0], ups[0])
    with pytest.raises(RuntimeError, match="outside"):
        _eager(api, scenes[1], ups[1])
    ref2 = _eager(api, scenes[2], ups[2])
    node = Node(api, 3, E, H, W, M, sub)
    node.write(scenes, ups)
    api.set_seed(999)
    node.both()                       # no exception
    assert node.fstatus.cpu().tolist() == [0, 1, 0] and node.bstatus.cpu().tolist() == [0, 1, 0]
    assert torch.isnan(node.scores[1]).all() and torch.isnan(node.poses[1]).all() and not node.contrib[1].any()
    np.testing.assert_array_equal(node.grads[1].cpu().numpy(), ups[1][2])   # untouched
    node.assert_eager(ref0, 0)
    node.assert_eager(ref2, 2)
    # a zeroed tape holds no forward: status 2, gradient untouched, the other images as before
    stride = api.hypotheses_tape_stride(E, H, W, M)
    node.tapes[:stride].zero_()
    node.grads.copy_(_cuda(np.stack([u[2] for u in ups])))
    node.backward()
    assert node.bstatus.cpu().tolist() == [2, 1, 0]
    np.testing.assert_array_equal(node.grads[0].cpu().numpy(), ups[0][2])
    np.testing.assert_array_equal(node.grads[1].cpu().numpy(), ups[1][2])
    np.testing.assert_array_equal(node.grads[2].cpu().numpy(), ref2[3])


def test_workspace_is_frozen_after_a_capture(api):
    import esac_b200.api as fresh_api
    E, H, W, M, sub = 2, 60, 80, 64, 8
    saved = fresh_api._contexts.get(0)
    ctx = fresh_api.Context(0)        # a context of its own: its workspace has seen only this test
    fresh_api._contexts[0] = ctx
    try:
        ctx.set_option("fixed_seed", 0)
        scenes = _scenes(3, E, H, W, M, sub, seed=800)
        ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
        fresh_api.reserve_backward_async(1, E, H, W, M, sub)
        node = Node(fresh_api, 1, E, H, W, M, sub)
        g = _capture(node.both)
        big = Node(fresh_api, 1, E, H, W, 4 * M, sub)
        big.scores.fill_(-1.0)
        with pytest.raises(RuntimeError, match="reserve_backward_async"):
            big.forward()
        with pytest.raises(RuntimeError, match="reserve_backward_async"):
            big.backward()
        assert (big.fstatus.cpu() == 7).all() and (big.bstatus.cpu() == 7).all()   # nothing was enqueued
        assert (big.scores.cpu() == -1.0).all()
        fresh_api.set_seed(31)
        ref = [_eager(fresh_api, sc, up) for sc, up in zip(scenes, ups)]
        fresh_api.set_seed(31)
        _replay_and_compare(g, node, scenes, ups, ref)
    finally:
        import torch
        torch.cuda.synchronize()
        if saved is not None:
            fresh_api._contexts[0] = saved
        else:
            fresh_api._contexts.pop(0, None)
        ctx.close()


def test_tapes_stay_independent_of_calls_in_between(api):
    E, H, W, M, sub = 3, 60, 80, 96, 8
    scenes = _scenes(2, E, H, W, M, sub, seed=850)
    ups = [_upstream(sc, k) for k, sc in enumerate(scenes)]
    ref = []
    for sc, up in zip(scenes, ups):
        api.set_seed(64)
        ref.append(_eager(api, sc, up))
    other = _scenes(1, 2, 30, 40, 48, 8, seed=860)[0]
    other_up = _upstream(other, 9)
    node = Node(api, 1, E, H, W, M, sub)
    small = Node(api, 1, 2, 30, 40, 48, 8)
    small.write([other], [other_up])
    for sc, up, r in zip(scenes, ups, ref):
        node.write([sc], [up])
        api.set_seed(64)
        node.forward()
        _eager(api, other, other_up)   # the eager node on another shape
        small.both()                   # the stream-ordered node on another shape
        node.backward()
        node.assert_eager(r)


class _StandIn:
    """Scene coordinates = a parameter map times a parameter scale, gating = log_softmax of a parameter row."""

    def __init__(self, sc, E):
        import torch
        self.coords = torch.nn.Parameter(_cuda(sc.coords))
        self.scale = torch.nn.Parameter(torch.ones((), device="cuda"))
        self.gate = torch.nn.Parameter(torch.linspace(-1.0, 1.0, E, device="cuda")[None])

    def params(self):
        return [self.coords, self.scale, self.gate]

    def __call__(self):
        import torch
        return self.coords * self.scale, torch.log_softmax(self.gate, 1)


def _dsac_star(T, gt):
    import torch
    cos = ((T[:, :3, :3] * gt[:3, :3]).sum((1, 2)) - 1) / 2
    angle = torch.rad2deg(torch.acos(cos.clamp(-1 + 1e-12, 1 - 1e-12)))
    return torch.maximum(angle, 100 * (T[:, :3, 3] - gt[:3, 3]).norm(dim=1))


def test_dsac_star_step_in_a_graph_equals_the_eager_step(api):
    import torch
    from esac_b200.autograd import esac_hypotheses, esac_hypotheses_async, pose_to_transform
    E, H, W, M, sub = 3, 60, 80, 128, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=900)
    net = _StandIn(scenes[0], E)
    assign = torch.zeros(M, dtype=torch.int64, device="cuda")
    gt = torch.zeros(4, 4, device="cuda")
    shift = torch.zeros(2, dtype=torch.int32, device="cuda")
    cam = torch.zeros(3, device="cuda")

    def write(sc):
        with torch.no_grad():
            net.coords.copy_(_cuda(sc.coords))
        assign.copy_(_cuda(sc.assign))
        gt.copy_(_cuda(sc.gt_pose))
        shift.copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
        cam.copy_(torch.tensor([sc.f, sc.ppx, sc.ppy]))

    def step(node):
        coords, glp = net()
        scores, poses, _ = node(coords)
        loss = (torch.softmax(scores, 0) * _dsac_star(pose_to_transform(poses), gt.double())).sum()
        counts = torch.zeros(E, device="cuda").scatter_add_(0, assign, torch.ones(M, device="cuda"))
        (loss + (loss.detach() * counts * glp[0]).sum()).backward()
        return loss.detach()

    def node_async(coords):
        return esac_hypotheses_async(coords, assign, shift, cam, *TAIL, sub)

    api.reserve_backward_async(1, E, H, W, M, sub)
    write(scenes[0])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(node_async)
    torch.cuda.current_stream().wait_stream(side)
    for p in net.params():
        p.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        loss = step(node_async)
    static_grads = [p.grad for p in net.params()]
    api.set_seed(2024)
    ref = []
    for sc in scenes:
        write(sc)
        for p in net.params():
            p.grad = None
        lo = step(lambda c: esac_hypotheses(c, assign, *sc.params))
        ref.append((lo.item(), [p.grad.clone() for p in net.params()]))
    api.set_seed(2024)
    for sc, (l_ref, g_ref) in zip(scenes, ref):
        write(sc)
        g.replay()
        assert loss.item() == l_ref
        for mine, gr in zip(static_grads, g_ref):
            assert torch.equal(mine, gr)
        assert torch.count_nonzero(static_grads[0]) > 0


def test_reference_loss_through_the_async_node_matches_backward_async(api):
    import torch
    from esac_b200.autograd import esac_hypotheses_async, reference_pose_loss_async
    E, H, W, M, sub = 3, 30, 40, 64, 8
    scenes = _scenes(2, E, H, W, M, sub, seed=950)
    assign = _cuda(np.stack([s.assign for s in scenes]))
    gts = _cuda(np.stack([s.gt_pose for s in scenes]))
    shifts = torch.tensor([[s.shiftX, s.shiftY] for s in scenes], dtype=torch.int32, device="cuda")
    cams = torch.tensor([[s.f, s.ppx, s.ppy] for s in scenes], device="cuda")
    coords = _cuda(np.stack([s.coords for s in scenes])).requires_grad_()
    api.set_seed(31337)
    scores, poses, _ = esac_hypotheses_async(coords, assign, shifts, cams, *TAIL, sub)
    mine = (torch.softmax(scores, 1) * reference_pose_loss_async(poses, gts, *LOSS)).sum(1)
    mine.sum().backward()
    losses = torch.zeros(2, dtype=torch.float64, device="cuda")
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    ref_grads = torch.zeros_like(coords)
    api.set_seed(31337)
    api.backward_async(coords.detach(), ref_grads, assign, gts, shifts, cams, *LOSS, *TAIL, sub, losses, status)
    assert (status.cpu() == 0).all()
    # the bars of the eager node's test: loss 1e-12 relative, gradient 1e-6 of the largest entry
    assert ((mine.detach() - losses).abs() <= 1e-12 * losses.abs()).all(), (mine, losses)
    for b in range(2):
        scale = ref_grads[b].abs().max().item()
        assert scale > 0 and (coords.grad[b] - ref_grads[b]).abs().max().item() <= 1e-6 * scale


def test_pose_loss_async_is_pose_loss_bitwise(api):
    import torch
    rng = np.random.default_rng(5)
    B, M = 3, 200
    poses = _cuda(np.concatenate([rng.standard_normal((B, M, 3)), rng.standard_normal((B, M, 3)) * 2], -1))
    scenes = _scenes(B, 1, 30, 40, 8, 8, seed=970)
    gts = _cuda(np.stack([s.gt_pose for s in scenes]))
    l_ref, d_ref = api.pose_loss(poses, gts, *LOSS)
    l, d = api.pose_loss_async(poses, gts, *LOSS)
    assert torch.equal(l, l_ref) and torch.equal(d, d_ref)
    l1, d1 = api.pose_loss_async(poses[1].contiguous(), gts[1].contiguous(), *LOSS)
    assert torch.equal(l1, l_ref[1]) and torch.equal(d1, d_ref[1])


def test_graph_example_checks_against_the_eager_step():
    import runpy
    import sys
    from pathlib import Path
    ex = Path(__file__).resolve().parents[1] / "examples" / "custom_loss_step_graph_synthetic.py"
    argv = sys.argv
    sys.argv = [str(ex), "--images", "3", "--check"]
    try:
        mod = runpy.run_path(str(ex), run_name="example")
        assert mod["main"]() == 0
    finally:
        sys.argv = argv
