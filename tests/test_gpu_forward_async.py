"""GPU tests of the stream-ordered forward (api.forward_async): bitwise equal to eager esac.forward call for call, a
captured CUDA graph that replays with new inputs, seeds and cameras, batches, no host synchronisation, the per-image
status, the workspace rule, and the graph example (run with `-m gpu`)."""
import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error

pytestmark = pytest.mark.gpu

TAIL = (10.0, 100.0, 0.5, 100.0)   # tau, alpha, beta, maxReproj


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 0)
    return api


def _scenes(n, E, H, W, M, sub, seed):
    """n images whose shift, focal length and principal point all differ."""
    out = []
    for k in range(n):
        f = 480.0 + 37.5 * k
        out.append(make_scene(E=E, H=H, W=W, M=M, sub=sub, seed=seed + k, f=f, ppx=W * sub / 2 + 3.25 * k - 4,
                              ppy=H * sub / 2 - 2.5 * k + 1, shiftX=k - 2, shiftY=1 - k))
    return out


def _eager(api, sc):
    import torch
    out = torch.zeros(4, 4, device="cuda")
    e = api.forward(torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda(), out, *sc.params)
    return out.cpu().numpy(), e


class Static:
    """The static inputs and outputs of a captured call, B images of one shape."""

    def __init__(self, B, E, H, W, M, sub):
        import torch
        self.sub = sub
        self.coords = torch.zeros(B, E, 3, H, W, device="cuda")
        self.assign = torch.zeros(B, M, dtype=torch.int64, device="cuda")
        self.shifts = torch.zeros(B, 2, dtype=torch.int32, device="cuda")
        self.cameras = torch.ones(B, 3, device="cuda")
        self.poses = torch.zeros(B, 4, 4, device="cuda")
        self.experts = torch.zeros(B, dtype=torch.int64, device="cuda")
        self.status = torch.zeros(B, dtype=torch.int32, device="cuda")

    def write(self, scenes):
        import torch
        for b, sc in enumerate(scenes):
            self.coords[b].copy_(torch.from_numpy(sc.coords))
            self.assign[b].copy_(torch.from_numpy(sc.assign))
            self.shifts[b].copy_(torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32))
            self.cameras[b].copy_(torch.tensor([sc.f, sc.ppx, sc.ppy], dtype=torch.float32))

    def call(self, api):
        api.forward_async(self.coords, self.assign, self.shifts, self.cameras, *TAIL, self.sub, self.poses, self.experts,
                          self.status)

    def results(self):
        return self.poses.cpu().numpy(), self.experts.cpu().numpy(), self.status.cpu().numpy()


def _capture(api, st):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st.call(api)
    return g


SHAPES = [  # E, H, W, M, sub
    (1, 60, 80, 64, 8),
    (7, 60, 80, 256, 8),
    (7, 480, 640, 256, 1),     # two sampling lanes, refinement over every co-resident CTA
    (2, 40, 27, 64, 8),        # portrait
    (3, 61, 107, 96, 8),       # N odd: scalar loads in the scoring kernel
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "E%d_%dx%d_M%d_sub%d" % s)
def test_calls_one_to_five_equal_eager_forward_bitwise(api, shape):
    import torch
    E, H, W, M, sub = shape
    scenes = _scenes(5, E, H, W, M, sub, seed=100 + E + H)
    api.set_seed(4242)
    ref = [_eager(api, sc) for sc in scenes]
    api.set_seed(4242)
    st = Static(1, E, H, W, M, sub)
    for sc, (pose, e) in zip(scenes, ref):
        st.write([sc])
        st.call(api)
        p, x, s = st.results()
        assert s[0] == 0
        assert x[0] == e
        np.testing.assert_array_equal(p[0], pose)
    # one image may also be passed unbatched
    api.set_seed(4242)
    sc = scenes[0]
    out, ex, stt = torch.zeros(4, 4, device="cuda"), torch.zeros((), dtype=torch.int64, device="cuda"), torch.zeros(
        (), dtype=torch.int32, device="cuda")
    api.forward_async(torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda(),
                      torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda"),
                      torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda"), *TAIL, sub, out, ex, stt)
    np.testing.assert_array_equal(out.cpu().numpy(), ref[0][0])
    assert int(ex) == ref[0][1] and int(stt) == 0


def _replay_and_compare(api, g, st, scenes, ref, between=None):
    for r, (sc, (pose, e)) in enumerate(zip(scenes, ref)):
        st.write([sc])
        if between:
            between(r)
        g.replay()
        p, x, s = st.results()
        assert s[0] == 0 and x[0] == e, (r, s, x, e)
        np.testing.assert_array_equal(p[0], pose)
        rot, trans = pose_error(p[0], sc.gt_pose)
        assert rot < 1.0 and trans < 0.05, (r, rot, trans)


def test_graph_replays_with_new_inputs_seeds_and_cameras(api):
    E, H, W, M, sub = 3, 60, 80, 64, 8
    scenes = _scenes(5, E, H, W, M, sub, seed=300)
    api.reserve_forward_async(1, E, H, W, M, sub)
    st = Static(1, E, H, W, M, sub)
    st.write([scenes[0]])
    g = _capture(api, st)
    # plain replays: replay r is eager call r
    api.set_seed(77)
    ref = [_eager(api, sc) for sc in scenes]
    api.set_seed(77)
    _replay_and_compare(api, g, st, scenes, ref)
    # set_seed between replays takes effect at the next replay
    api.set_seed(78)
    ref = [_eager(api, sc) for sc in scenes[:2]]
    api.set_seed(91)
    ref += [_eager(api, sc) for sc in scenes[2:]]
    api.set_seed(78)
    _replay_and_compare(api, g, st, scenes, ref, between=lambda r: api.set_seed(91) if r == 2 else None)
    # eager calls of other shapes between replays leave the graph's buffers alone
    other = make_scene(E=5, H=90, W=120, M=300, sub=8, seed=5)
    api.set_seed(79)
    ref = [_eager(api, sc) for sc in scenes]
    api.set_seed(79)
    _replay_and_compare(api, g, st, scenes, ref, between=lambda r: _eager(api, other))


def test_graph_with_fixed_seed(api):
    E, H, W, M, sub = 2, 60, 80, 64, 8
    scenes = _scenes(4, E, H, W, M, sub, seed=400)
    api.reserve_forward_async(1, E, H, W, M, sub)
    ctx = api.context()
    ctx.set_option("fixed_seed", 1)
    try:
        st = Static(1, E, H, W, M, sub)
        g = _capture(api, st)
        api.set_seed(123)
        ref = [_eager(api, sc) for sc in scenes]
        api.set_seed(123)
        _replay_and_compare(api, g, st, scenes, ref)
    finally:
        ctx.set_option("fixed_seed", 0)


def test_batch_equals_forward_batch_with_per_image_arrays(api):
    import torch
    E, H, W, M, sub = 3, 30, 40, 48, 8
    scenes = _scenes(4, E, H, W, M, sub, seed=500)
    coords = torch.from_numpy(np.stack([s.coords for s in scenes])).cuda()
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    cams = ([s.shiftX for s in scenes], [s.shiftY for s in scenes], [s.f for s in scenes], [s.ppx for s in scenes],
            [s.ppy for s in scenes])
    api.set_seed(555)
    refs = []
    for _ in range(2):   # eager calls 0..3, then 4..7
        out = torch.zeros(4, 4, 4, device="cuda")
        e = api.forward_batch(coords, assign, out, *cams, *TAIL, sub)
        refs.append((out.cpu().numpy(), e))
    st = Static(4, E, H, W, M, sub)
    st.write(scenes)
    api.set_seed(555)
    st.call(api)
    p, x, s = st.results()
    assert (s == 0).all() and list(x) == refs[0][1]
    np.testing.assert_array_equal(p, refs[0][0])
    api.reserve_forward_async(4, E, H, W, M, sub)
    g = _capture(api, st)
    st.poses.zero_()
    api.set_seed(555)
    for ref_p, ref_e in refs:   # replay j is the j-th execution: images 4j .. 4j + 3 of the eager sequence
        g.replay()
        p, x, s = st.results()
        assert (s == 0).all() and list(x) == ref_e
        np.testing.assert_array_equal(p, ref_p)


def test_no_host_synchronisation(api):
    import torch
    E, H, W, M, sub = 2, 60, 80, 64, 8
    sc = _scenes(1, E, H, W, M, sub, seed=600)[0]
    api.reserve_forward_async(1, E, H, W, M, sub)
    st = Static(1, E, H, W, M, sub)
    st.write([sc])
    st.call(api)                      # first call: nothing left to set up
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(int(2e9))       # ~1 s of device time ahead of the call
    st.call(api)
    assert not stream.query(), "forward_async waited for the device"
    torch.cuda.synchronize()
    # capture in torch's default (global) error mode, with torch work before and after the call in the same graph
    g = torch.cuda.CUDAGraph()
    src = st.coords.clone()
    doubled = torch.zeros_like(st.poses)
    with torch.cuda.graph(g):
        st.coords.copy_(src * 1.0)
        st.call(api)
        doubled.copy_(st.poses * 2.0)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))
    g.replay()
    assert not stream.query(), "graph.replay() waited for the device"
    torch.cuda.synchronize()
    p, _, s = st.results()
    assert s[0] == 0
    np.testing.assert_array_equal(doubled.cpu().numpy(), 2.0 * p)


def test_bad_expert_index_sets_the_status_of_that_image_only(api):
    E, H, W, M, sub = 3, 30, 40, 48, 8
    scenes = _scenes(3, E, H, W, M, sub, seed=700)
    scenes[1].assign[5] = E   # outside [0, E)
    api.set_seed(999)
    ref0 = _eager(api, scenes[0])
    with pytest.raises(RuntimeError, match="outside"):
        _eager(api, scenes[1])
    ref2 = _eager(api, scenes[2])
    st = Static(3, E, H, W, M, sub)
    st.write(scenes)
    api.set_seed(999)
    st.call(api)                      # no exception
    p, x, s = st.results()
    assert list(s) == [0, 1, 0]
    assert list(x) == [ref0[1], -1, ref2[1]]
    assert np.isnan(p[1]).all()
    np.testing.assert_array_equal(p[0], ref0[0])
    np.testing.assert_array_equal(p[2], ref2[0])


def test_workspace_is_frozen_after_a_capture(api):
    import esac_b200.api as fresh_api
    E, H, W, M, sub = 2, 60, 80, 64, 8
    ctx = fresh_api.Context(0)        # a context of its own: its workspace has seen only this test
    saved = fresh_api._contexts.get(0)
    fresh_api._contexts[0] = ctx
    try:
        scenes = _scenes(3, E, H, W, M, sub, seed=800)
        fresh_api.reserve_forward_async(1, E, H, W, M, sub)
        st = Static(1, E, H, W, M, sub)
        g = _capture(fresh_api, st)
        big = Static(1, E, H, W, 4 * M, sub)
        big.status.fill_(7)
        with pytest.raises(RuntimeError, match="reserve_forward_async"):
            big.call(fresh_api)
        assert int(big.status.item()) == 7          # nothing was enqueued
        with pytest.raises(RuntimeError, match="reserve_forward_async"):
            fresh_api.reserve_forward_async(1, E, 2 * H, W, M, sub)
        fresh_api.reserve_forward_async(1, E, H, W, M // 2, sub)   # smaller fits
        fresh_api.set_seed(31)
        ref = [_eager(fresh_api, sc) for sc in scenes]
        fresh_api.set_seed(31)
        _replay_and_compare(fresh_api, g, st, scenes, ref)
    finally:
        if saved is not None:
            fresh_api._contexts[0] = saved
        else:
            fresh_api._contexts.pop(0, None)
        ctx.close()


def test_graph_example_checks_against_eager_forward():
    import runpy
    import sys
    from pathlib import Path
    ex = Path(__file__).resolve().parents[1] / "examples" / "test_step_graph_synthetic.py"
    argv = sys.argv
    sys.argv = [str(ex), "--images", "4", "--check"]
    try:
        mod = runpy.run_path(str(ex), run_name="example")
        assert mod["main"]() == 0
    finally:
        sys.argv = argv
