"""GPU tests of the stream-ordered backward (api.backward_async) and its autograd node (autograd.esac_loss_async): bitwise
equal to eager esac.backward call for call, a captured CUDA graph that replays with new inputs, ground truths, seeds and
cameras and picks its refinement group on the device, one call counter with forward_async, batches, no host
synchronisation, the per-image status, the workspace rule, a captured training step, and the graph example (run with
`-m gpu`)."""
import numpy as np
import pytest

from esac_b200.synth import make_scene

pytestmark = pytest.mark.gpu

LOSS = (1.0, 100.0, 100.0)          # wLossRot, wLossTrans, lossCut
TAIL = (10.0, 100.0, 0.5, 100.0)    # tau, alpha, beta, maxReproj

SHAPES = [  # E, H, W, M, sub: the shapes of test_gpu_forward_async.py
    (1, 60, 80, 64, 8),
    (7, 60, 80, 256, 8),
    (7, 480, 640, 256, 1),     # two sampling lanes, refinement groups of many CTAs
    (2, 40, 27, 64, 8),        # portrait
    (3, 61, 107, 96, 8),       # N odd
]


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 0)
    return api


def _scenes(n, E, H, W, M, sub, seed, **kw):
    """n images whose shift, focal length, principal point and ground truth all differ."""
    out = []
    for k in range(n):
        f = 480.0 + 37.5 * k
        out.append(make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=seed + k, f=f, ppx=W * sub / 2 + 3.25 * k - 4,
                              ppy=H * sub / 2 - 2.5 * k + 1, shiftX=k - 2, shiftY=1 - k, **kw))
    return out


def _grads0(sc, k):
    """A non-zero starting gradient: both entry points accumulate (+=)."""
    return np.random.default_rng(1000 + k).standard_normal(sc.coords.shape).astype(np.float32) * 1e-3


def _eager(api, sc, g0):
    """esac.backward on device tensors (device ground truth); returns (loss, gradient, refinement group)."""
    import torch
    grads = torch.from_numpy(g0.copy()).cuda()
    loss = api.backward(torch.from_numpy(sc.coords).cuda(), grads, torch.from_numpy(sc.assign).cuda(),
                        torch.from_numpy(sc.gt_pose).cuda(), *LOSS, *sc.params)
    return loss, grads.cpu().numpy(), api.last_stats()["refine_group"]


class Static:
    """The static inputs and outputs of a captured call, B images of one shape."""

    def __init__(self, B, E, H, W, M, sub):
        import torch
        self.sub = sub
        self.coords = torch.zeros(B, E, 3, H, W, device="cuda")
        self.grads = torch.zeros(B, E, 3, H, W, device="cuda")
        self.assign = torch.zeros(B, M, dtype=torch.int64, device="cuda")
        self.gt = torch.eye(4, device="cuda").repeat(B, 1, 1)
        self.shifts = torch.zeros(B, 2, dtype=torch.int32, device="cuda")
        self.cameras = torch.ones(B, 3, device="cuda")
        self.losses = torch.zeros(B, dtype=torch.float64, device="cuda")
        self.status = torch.zeros(B, dtype=torch.int32, device="cuda")

    def write(self, scenes, g0s):
        import torch
        for b, (sc, g0) in enumerate(zip(scenes, g0s)):
            self.coords[b].copy_(torch.from_numpy(sc.coords))
            self.grads[b].copy_(torch.from_numpy(g0))
            self.assign[b].copy_(torch.from_numpy(sc.assign))
            self.gt[b].copy_(torch.from_numpy(sc.gt_pose))
            self.shifts[b].copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
            self.cameras[b].copy_(torch.tensor([sc.f, sc.ppx, sc.ppy], dtype=torch.float32))

    def call(self, api):
        api.backward_async(self.coords, self.grads, self.assign, self.gt, self.shifts, self.cameras, *LOSS, *TAIL, self.sub,
                           self.losses, self.status)

    def results(self):
        return self.losses.cpu().numpy(), self.grads.cpu().numpy(), self.status.cpu().numpy()


def _capture(api, st):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st.call(api)
    return g


def _assert_same(loss, grads, ref):
    assert np.float64(loss) == np.float64(ref[0]), (loss, ref[0])
    np.testing.assert_array_equal(grads, ref[1])


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "E%d_%dx%d_M%d_sub%d" % s)
def test_calls_one_to_five_equal_eager_backward_bitwise(api, shape):
    import torch
    E, H, W, M, sub = shape
    scenes = _scenes(5, E, H, W, M, sub, seed=100 + E + H)
    g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
    api.set_seed(4242)
    ref = [_eager(api, sc, g0) for sc, g0 in zip(scenes, g0s)]
    api.set_seed(4242)
    st = Static(1, E, H, W, M, sub)
    for sc, g0, r in zip(scenes, g0s, ref):
        st.write([sc], [g0])
        st.call(api)
        lo, gr, s = st.results()
        assert s[0] == 0
        _assert_same(lo[0], gr[0], r)
    # one image may also be passed unbatched
    api.set_seed(4242)
    sc = scenes[0]
    grads = torch.from_numpy(g0s[0].copy()).cuda()
    lo, stt = torch.zeros((), dtype=torch.float64, device="cuda"), torch.zeros((), dtype=torch.int32, device="cuda")
    api.backward_async(torch.from_numpy(sc.coords).cuda(), grads, torch.from_numpy(sc.assign).cuda(),
                       torch.from_numpy(sc.gt_pose).cuda(), torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda"),
                       torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda"), *LOSS, *TAIL, sub, lo, stt)
    assert int(stt) == 0
    _assert_same(float(lo), grads.cpu().numpy(), ref[0])


def _replay_and_compare(g, st, scenes, g0s, ref, between=None):
    for r, (sc, g0, rf) in enumerate(zip(scenes, g0s, ref)):
        st.write([sc], [g0])
        if between:
            between(r)
        g.replay()
        lo, gr, s = st.results()
        assert s[0] == 0, (r, s)
        _assert_same(lo[0], gr[0], rf)


def _varied_scenes(E, H, W, M, sub):
    """Scenes from clean to mostly outliers: the number of contributing hypotheses, and with it the refinement group
    esac.backward picks, differs between them."""
    out = []
    for k, (frac, noise) in enumerate([(0.4, 0.02), (0.9, 0.3), (0.1, 0.005), (0.8, 0.15), (0.95, 0.5), (0.6, 0.05)]):
        f = 500.0 + 40.0 * k
        out.append(make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=300 + k, f=f, ppx=W * sub / 2 + k, ppy=H * sub / 2 - k,
                              shiftX=2 - k, shiftY=k - 3, outlier_frac=frac, noise=noise))
    return out


def test_graph_replays_with_new_inputs_seeds_and_cameras(api):
    E, H, W, M, sub = 3, 60, 80, 256, 8
    scenes = _varied_scenes(E, H, W, M, sub)
    g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
    api.reserve_backward_async(1, E, H, W, M, sub)
    st = Static(1, E, H, W, M, sub)
    st.write([scenes[0]], [g0s[0]])
    api.set_seed(77)
    g = _capture(api, st)
    # plain replays: replay r is eager call r, whatever refinement group its contributing hypotheses call for
    api.set_seed(77)
    ref = [_eager(api, sc, g0) for sc, g0 in zip(scenes, g0s)]
    groups = [r[2] for r in ref]
    assert len(set(groups)) >= 2, groups   # the device picks the group per replay: it is not frozen at capture
    api.set_seed(77)
    _replay_and_compare(g, st, scenes, g0s, ref)
    # set_seed between replays takes effect at the next replay
    api.set_seed(78)
    ref = [_eager(api, sc, g0) for sc, g0 in zip(scenes[:2], g0s[:2])]
    api.set_seed(91)
    ref += [_eager(api, sc, g0) for sc, g0 in zip(scenes[2:], g0s[2:])]
    api.set_seed(78)
    _replay_and_compare(g, st, scenes, g0s, ref, between=lambda r: api.set_seed(91) if r == 2 else None)
    # eager calls of other shapes between replays leave the graph's buffers alone
    other = make_scene(E=5, H=90, W=120, M=300, sub=8, seed=5)
    api.set_seed(79)
    ref = [_eager(api, sc, g0) for sc, g0 in zip(scenes, g0s)]
    api.set_seed(79)
    _replay_and_compare(g, st, scenes, g0s, ref, between=lambda r: _eager(api, other, np.zeros_like(other.coords)))


def test_graph_with_fixed_seed(api):
    E, H, W, M, sub = 2, 60, 80, 64, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=400)
    g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
    api.reserve_backward_async(1, E, H, W, M, sub)
    ctx = api.context()
    ctx.set_option("fixed_seed", 1)
    try:
        st = Static(1, E, H, W, M, sub)
        g = _capture(api, st)
        api.set_seed(123)
        ref = [_eager(api, sc, g0) for sc, g0 in zip(scenes, g0s)]
        api.set_seed(123)
        _replay_and_compare(g, st, scenes, g0s, ref)
    finally:
        ctx.set_option("fixed_seed", 0)


def test_forward_and_backward_in_one_graph_share_the_call_counter(api):
    import torch
    E, H, W, M, sub = 3, 60, 80, 64, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=450)
    g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
    api.reserve_backward_async(1, E, H, W, M, sub)
    st = Static(1, E, H, W, M, sub)
    pose = torch.zeros(1, 4, 4, device="cuda")
    expert = torch.zeros(1, dtype=torch.int64, device="cuda")
    fstatus = torch.zeros(1, dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        api.forward_async(st.coords, st.assign, st.shifts, st.cameras, *TAIL, sub, pose, expert, fstatus)
        st.call(api)
    api.set_seed(5150)
    ref = []
    for sc, g0 in zip(scenes, g0s):   # eager: forward (call 2r), then backward (call 2r + 1)
        out = torch.zeros(4, 4, device="cuda")
        e = api.forward(torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda(), out, *sc.params)
        ref.append((out.cpu().numpy(), e) + _eager(api, sc, g0))
    api.set_seed(5150)
    for sc, g0, (p_ref, e_ref, l_ref, g_ref, _) in zip(scenes, g0s, ref):
        st.write([sc], [g0])
        g.replay()
        lo, gr, s = st.results()
        assert s[0] == 0 and int(fstatus[0]) == 0
        assert int(expert[0]) == e_ref
        np.testing.assert_array_equal(pose[0].cpu().numpy(), p_ref)
        _assert_same(lo[0], gr[0], (l_ref, g_ref))


def test_batch_equals_backward_batch_with_per_image_arrays(api):
    import torch
    E, H, W, M, sub = 3, 30, 40, 48, 8
    scenes = _scenes(4, E, H, W, M, sub, seed=500)
    g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
    coords = torch.from_numpy(np.stack([s.coords for s in scenes])).cuda()
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    cams = ([s.shiftX for s in scenes], [s.shiftY for s in scenes], [s.f for s in scenes], [s.ppx for s in scenes],
            [s.ppy for s in scenes])
    api.set_seed(555)
    refs = []
    for _ in range(2):   # eager calls 0..3, then 4..7
        grads = torch.from_numpy(np.stack(g0s)).cuda()
        losses = api.backward_batch(coords, grads, assign, gts, *LOSS, *cams, *TAIL, sub)
        refs.append((np.array(losses), grads.cpu().numpy()))
    st = Static(4, E, H, W, M, sub)
    st.write(scenes, g0s)
    api.set_seed(555)
    st.call(api)
    lo, gr, s = st.results()
    assert (s == 0).all()
    np.testing.assert_array_equal(lo, refs[0][0])
    np.testing.assert_array_equal(gr, refs[0][1])
    api.reserve_backward_async(4, E, H, W, M, sub)
    g = _capture(api, st)
    api.set_seed(555)
    for ref_l, ref_g in refs:   # replay j is the j-th execution: images 4j .. 4j + 3 of the eager sequence
        st.grads.copy_(torch.from_numpy(np.stack(g0s)))
        g.replay()
        lo, gr, s = st.results()
        assert (s == 0).all()
        np.testing.assert_array_equal(lo, ref_l)
        np.testing.assert_array_equal(gr, ref_g)


def test_no_host_synchronisation(api):
    import torch
    E, H, W, M, sub = 2, 60, 80, 64, 8
    sc = _scenes(1, E, H, W, M, sub, seed=600)[0]
    api.reserve_backward_async(1, E, H, W, M, sub)
    st = Static(1, E, H, W, M, sub)
    st.write([sc], [np.zeros_like(sc.coords)])
    st.call(api)                      # first call: nothing left to set up
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(int(2e9))       # ~1 s of device time ahead of the call
    st.call(api)
    assert not stream.query(), "backward_async waited for the device"
    torch.cuda.synchronize()
    # capture in torch's default (global) error mode, with torch work before and after the call in the same graph
    g = torch.cuda.CUDAGraph()
    src = st.coords.clone()
    doubled = torch.zeros_like(st.losses)
    with torch.cuda.graph(g):
        st.coords.copy_(src * 1.0)
        st.grads.zero_()
        st.call(api)
        doubled.copy_(st.losses * 2.0)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))
    g.replay()
    assert not stream.query(), "graph.replay() waited for the device"
    torch.cuda.synchronize()
    lo, _, s = st.results()
    assert s[0] == 0 and np.isfinite(lo[0])
    np.testing.assert_array_equal(doubled.cpu().numpy(), 2.0 * lo)


def test_bad_expert_index_sets_the_status_of_that_image_only(api):
    E, H, W, M, sub = 3, 30, 40, 48, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=700)
    g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
    scenes[1].assign[5] = E   # outside [0, E)
    api.set_seed(999)
    ref0 = _eager(api, scenes[0], g0s[0])
    with pytest.raises(RuntimeError, match="outside"):
        _eager(api, scenes[1], g0s[1])
    ref2 = _eager(api, scenes[2], g0s[2])
    st = Static(3, E, H, W, M, sub)
    st.write(scenes, g0s)
    api.set_seed(999)
    st.call(api)                      # no exception
    lo, gr, s = st.results()
    assert list(s) == [0, 1, 0]
    assert np.isnan(lo[1])
    np.testing.assert_array_equal(gr[1], g0s[1])   # untouched
    _assert_same(lo[0], gr[0], ref0)
    _assert_same(lo[2], gr[2], ref2)


def test_workspace_is_frozen_after_a_capture(api):
    import esac_b200.api as fresh_api
    E, H, W, M, sub = 2, 60, 80, 64, 8
    ctx = fresh_api.Context(0)        # a context of its own: its workspace has seen only this test
    saved = fresh_api._contexts.get(0)
    fresh_api._contexts[0] = ctx
    try:
        scenes = _scenes(3, E, H, W, M, sub, seed=800)
        g0s = [_grads0(sc, k) for k, sc in enumerate(scenes)]
        fresh_api.reserve_backward_async(1, E, H, W, M, sub)
        st = Static(1, E, H, W, M, sub)
        g = _capture(fresh_api, st)
        big = Static(1, E, H, W, 4 * M, sub)
        big.status.fill_(7)
        big.losses.fill_(-1.0)
        with pytest.raises(RuntimeError, match="reserve_backward_async"):
            big.call(fresh_api)
        assert int(big.status.item()) == 7 and float(big.losses.item()) == -1.0   # nothing was enqueued
        with pytest.raises(RuntimeError, match="reserve_backward_async"):
            fresh_api.reserve_backward_async(1, E, 2 * H, W, M, sub)
        fresh_api.reserve_backward_async(1, E, H, W, M // 2, sub)   # smaller fits
        fresh_api.set_seed(31)
        ref = [_eager(fresh_api, sc, g0) for sc, g0 in zip(scenes, g0s)]
        fresh_api.set_seed(31)
        _replay_and_compare(g, st, scenes, g0s, ref)
    finally:
        if saved is not None:
            fresh_api._contexts[0] = saved
        else:
            fresh_api._contexts.pop(0, None)
        ctx.close()


class _StandIn:
    """A stand-in network: scene coordinates = a parameter map times a parameter scale, gating = log_softmax of a parameter
    row, so that the gradients of both outputs land in parameters through torch's own backward."""

    def __init__(self, sc, E):
        import torch
        self.coords = torch.nn.Parameter(torch.from_numpy(sc.coords).cuda())
        self.scale = torch.nn.Parameter(torch.ones((), device="cuda"))
        self.gate = torch.nn.Parameter(torch.linspace(-1.0, 1.0, E, device="cuda")[None])

    def params(self):
        return [self.coords, self.scale, self.gate]

    def __call__(self):
        import torch
        return self.coords * self.scale, torch.log_softmax(self.gate, 1)


@pytest.mark.parametrize("expert_selection", [False, True])
def test_esac_loss_async_in_a_graph_equals_esac_loss(api, expert_selection):
    import torch
    from esac_b200.autograd import esac_loss, esac_loss_async
    E, H, W, M, sub = 3, 60, 80, 128, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=900)
    net = _StandIn(scenes[0], E)
    assign = torch.zeros(M, dtype=torch.int64, device="cuda")
    drawn = torch.zeros(1, dtype=torch.int64, device="cuda")
    hyp = drawn.expand(M) if expert_selection else assign       # expert.expand(M), train_esac.py:133-135
    gt = torch.zeros(4, 4, device="cuda")
    shift = torch.zeros(2, dtype=torch.int32, device="cuda")
    cam = torch.zeros(3, device="cuda")

    def write(sc):
        with torch.no_grad():
            net.coords.copy_(torch.from_numpy(sc.coords))
        assign.copy_(torch.from_numpy(sc.assign))
        drawn.fill_(int(sc.assign[0]))
        gt.copy_(torch.from_numpy(sc.gt_pose))
        shift.copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
        cam.copy_(torch.tensor([sc.f, sc.ppx, sc.ppy]))

    def step():
        coords, glp = net()
        loss = esac_loss_async(coords, glp, hyp, gt, shift, cam, *LOSS, *TAIL, sub, expert_selection=expert_selection)
        loss.backward()
        return loss.detach()

    api.reserve_backward_async(1, E, H, W, M, sub)
    write(scenes[0])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    for p in net.params():
        p.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        loss = step()
    static_grads = [p.grad for p in net.params()]   # the graph's gradient buffers
    api.set_seed(2024)
    ref = []
    for sc in scenes:   # eager esac_loss on the same parameters: loss and every parameter's gradient
        write(sc)
        for p in net.params():
            p.grad = None
        coords, glp = net()
        lo = esac_loss(coords, glp, hyp, gt, *LOSS, sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy, *TAIL, sub,
                       expert_selection=expert_selection)
        lo.backward()
        ref.append((lo.item(), [p.grad.clone() for p in net.params()]))
    api.set_seed(2024)
    for sc, (l_ref, g_ref) in zip(scenes, ref):
        write(sc)
        g.replay()
        assert loss.dtype == torch.float32 and loss.item() == l_ref
        for mine, gr in zip(static_grads, g_ref):
            assert torch.equal(mine, gr)
        assert torch.count_nonzero(static_grads[2]) > 0


def test_esac_loss_async_batch_equals_esac_loss_batch(api):
    import torch
    from esac_b200.autograd import esac_loss_async, esac_loss_batch
    E, H, W, M, sub = 3, 30, 40, 64, 8
    scenes = _scenes(2, E, H, W, M, sub, seed=950)
    coords = torch.from_numpy(np.stack([s.coords for s in scenes])).cuda().requires_grad_()
    gate = torch.randn(2, E, device="cuda", requires_grad=True)
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    shifts = torch.tensor([[s.shiftX, s.shiftY] for s in scenes], dtype=torch.int32, device="cuda")
    cams = torch.tensor([[s.f, s.ppx, s.ppy] for s in scenes], device="cuda")
    upstream = torch.tensor([0.75, -1.5], device="cuda")
    api.set_seed(31337)
    ref = esac_loss_batch(coords, torch.log_softmax(gate, 1), assign, gts, *LOSS, list(shifts[:, 0].tolist()),
                          list(shifts[:, 1].tolist()), [s.f for s in scenes], [s.ppx for s in scenes], [s.ppy for s in scenes],
                          *TAIL, sub)
    (ref * upstream).sum().backward()
    ref_grads = coords.grad.clone(), gate.grad.clone()
    coords.grad = gate.grad = None
    api.set_seed(31337)
    out = esac_loss_async(coords, torch.log_softmax(gate, 1), assign, gts, shifts, cams, *LOSS, *TAIL, sub)
    (out * upstream).sum().backward()
    assert torch.equal(out, ref)
    assert torch.equal(coords.grad, ref_grads[0]) and torch.equal(gate.grad, ref_grads[1])


def test_graph_example_checks_against_eager_backward():
    import runpy
    import sys
    from pathlib import Path
    ex = Path(__file__).resolve().parents[1] / "examples" / "train_step_graph_synthetic.py"
    argv = sys.argv
    sys.argv = [str(ex), "--images", "4", "--check"]
    try:
        mod = runpy.run_path(str(ex), run_name="example")
        assert mod["main"]() == 0
    finally:
        sys.argv = argv
