"""GPU tests of the stream-ordered losses (api.reproj_loss_async / coord_loss_async / reserve_loss_async and
autograd.reproj_loss_async / coord_loss_async): bitwise equal to the eager calls, graph replays with new maps, ground
truths, pads and cameras (the device inversion of the ground truth rounds as the host's), the per-image status of a
singular ground truth, no host synchronisation, the workspace rule, captured training steps and the two graph examples
(run with `-m gpu`)."""
import math

import numpy as np
import pytest

from orientations import NAMES, ORIENTATIONS, cam_to_world, rotate, uniform_rotations

pytestmark = pytest.mark.gpu

CUT, MAXR, MIND = 10.0, 100.0, 0.1


@pytest.fixture(scope="module")
def api():
    """The module's own context, so that the stream-ordered workspace here has seen only these tests."""
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


def _rotations():
    return ([ORIENTATIONS[k] for k in NAMES] + uniform_rotations(8, 2024) +
            [rotate(ORIENTATIONS["identity"], (1.0, 1.0, 0.0), math.pi - 1e-6)])


def _gt_poses(n, seed, first=None):
    """n camera->world ground truths, j = first .. first + n - 1: rotation j of tests/orientations.py's set, uniform ones
    and one near pi, cycled; every fifth an ill-conditioned block (one axis scaled by 1e-4, and a shear)."""
    rots = _rotations()
    rng = np.random.default_rng(seed)
    first = 7 * seed if first is None else first
    out = []
    for j in range(first, first + n):
        T = cam_to_world(rots[j % len(rots)], rng.uniform(-2.0, 2.0, 3)).astype(np.float64)
        if j % 5 == 4:
            T[:3, :3] = T[:3, :3] @ np.diag([1.0, 1e-4, 1.0]) + 1e-3 * rng.standard_normal((3, 3))
        out.append(T.astype(np.float32))
    return np.stack(out)


def _reproj_inputs(shapes, sub, seed, first=None):
    """Predictions in front of each camera (depth 1-6 m) with a few cells behind it, ground truths (_gt_poses), pads and
    cameras."""
    import torch
    rng = np.random.default_rng(seed)
    gts = _gt_poses(len(shapes), seed, first)
    preds = []
    for (H, W), T in zip(shapes, gts):
        z = rng.uniform(1.0, 6.0, (H, W))
        z[rng.random((H, W)) < 0.03] = -0.5
        x = (rng.random((H, W)) - 0.5) * z
        y = (rng.random((H, W)) - 0.5) * z
        cam = np.stack([x, y, z, np.ones_like(z)]).reshape(4, -1)
        world = (T.astype(np.float64) @ cam)[:3].reshape(3, H, W)
        preds.append(torch.from_numpy(world.astype(np.float32)).cuda())
    shifts = torch.from_numpy(rng.integers(-4, 5, (len(shapes), 2)).astype(np.int32)).cuda()
    cams = torch.from_numpy(np.stack([[rng.uniform(400, 600), W * sub / 2 + rng.uniform(-5, 5), H * sub / 2 + rng.uniform(-5, 5)]
                                      for H, W in shapes]).astype(np.float32)).cuda()
    return preds, torch.from_numpy(gts).cuda(), shifts, cams


def _reproj_eager(api, pred, gts, shifts, cams, sub, grads=None):
    s, c = shifts.cpu().numpy(), cams.cpu().numpy()
    return api.reproj_loss(pred, gts, c[:, 0], s[:, 0], s[:, 1], CUT, sub, c[:, 1], c[:, 2], outGradients=grads,
                           maxReproj=MAXR, minDepth=MIND)


def _reproj_async(api, pred, gts, shifts, cams, sub, grads=None):
    import torch
    B = len(pred) if isinstance(pred, list) else pred.shape[0]
    losses = torch.full((B,), -1.0, dtype=torch.float64, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    api.reproj_loss_async(pred, gts, shifts, cams, CUT, sub, losses, status, outGradients=grads, maxReproj=MAXR, minDepth=MIND)
    return losses, status


def _equal(a, b):
    """Bitwise, NaN included."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


REPROJ_CASES = [((60, 80), 8, 1), ((60, 80), 8, 4), ((480, 640), 1, 1), ((480, 640), 1, 4)]


@pytest.mark.parametrize("shape,sub,B", REPROJ_CASES, ids=lambda v: str(v))
def test_reproj_uncaptured_equals_eager_bitwise(api, shape, sub, B):
    import torch
    preds, gts, shifts, cams = _reproj_inputs([shape] * B, sub, seed=B + shape[0])
    pred = torch.stack(preds)
    g_ref, g = torch.zeros_like(pred), torch.full_like(pred, 7.0)
    ref = _reproj_eager(api, pred, gts, shifts, cams, sub, g_ref)
    losses, status = _reproj_async(api, pred, gts, shifts, cams, sub, g)
    assert _equal(losses.cpu().numpy(), np.array(ref)) and status.tolist() == [0] * B
    assert _equal(g.cpu().numpy(), g_ref.cpu().numpy())
    # loss only
    losses, status = _reproj_async(api, pred, gts, shifts, cams, sub)
    assert _equal(losses.cpu().numpy(), np.array(ref))


def test_reproj_ragged_and_misaligned(api):
    import torch
    shapes = [(60, 80), (7, 5), (45, 61), (30, 3), (480, 640)]
    preds, gts, shifts, cams = _reproj_inputs(shapes, 8, seed=5)
    # image 2 a misaligned view (the scalar load path), the others contiguous
    base = torch.empty(3 * 45 * 61 + 1, device="cuda")
    preds[2] = base[1:].view(3, 45, 61).copy_(preds[2])
    grads = [torch.zeros_like(p) for p in preds]
    g_ref = [torch.zeros_like(p) for p in preds]
    ref = _reproj_eager(api, preds, gts, shifts, cams, 8, g_ref)
    losses, status = _reproj_async(api, preds, gts, shifts, cams, 8, grads)
    assert _equal(losses.cpu().numpy(), np.array(ref)) and status.tolist() == [0] * 5
    for a, b in zip(grads, g_ref):
        assert _equal(a.cpu().numpy(), b.cpu().numpy())
    # a misaligned stacked view
    flat = torch.empty(2 * 3 * 60 * 80 + 1, device="cuda")
    pred = flat[1:].view(2, 3, 60, 80).copy_(torch.stack([preds[0], preds[0] * 1.01]))
    gflat = torch.zeros(2 * 3 * 60 * 80 + 3, device="cuda")
    g = gflat[3:].view(2, 3, 60, 80)
    g_ref = torch.zeros(2, 3, 60, 80, device="cuda")
    ref = _reproj_eager(api, pred, gts[:2].contiguous(), shifts[:2].contiguous(), cams[:2].contiguous(), 8, g_ref)
    losses, _ = _reproj_async(api, pred, gts[:2].contiguous(), shifts[:2].contiguous(), cams[:2].contiguous(), 8, g)
    assert _equal(losses.cpu().numpy(), np.array(ref)) and _equal(g.cpu().numpy(), g_ref.cpu().numpy())


def _coord_inputs(shapes, seed, bigger=False, empty=()):
    """Predictions (one cell larger than the ground truth when `bigger`) around ground truths with a third of the cells
    invalid and errors on both sides of the cut; images in `empty` have no valid cell."""
    import torch
    rng = np.random.default_rng(seed)
    preds, gts = [], []
    for b, (H, W) in enumerate(shapes):
        q = rng.uniform(-5, 5, (3, H, W)).astype(np.float32)
        q[:, rng.random((H, W)) < 0.33] = 0.0
        if b in empty:
            q[:] = 0.0
        hp, wp = (H + 1, W + 1) if bigger else (H, W)
        p = rng.standard_normal((3, hp, wp)) * 10.0 ** rng.uniform(-2, 3, (1, hp, wp))
        p[:, :H, :W] += q
        preds.append(torch.from_numpy(p.astype(np.float32)).cuda())
        gts.append(torch.from_numpy(q).cuda())
    return preds, gts


def _coord_async(api, pred, gt, grads=None, counts=True):
    import torch
    B = len(pred) if isinstance(pred, list) else pred.shape[0]
    losses = torch.full((B,), -1.0, dtype=torch.float64, device="cuda")
    cnt = torch.full((B,), -1, dtype=torch.int64, device="cuda") if counts else None
    api.coord_loss_async(pred, gt, CUT, losses, outGradients=grads, outCounts=cnt)
    return losses, cnt


@pytest.mark.parametrize("shape,B", [((60, 80), 1), ((60, 80), 4), ((480, 640), 1), ((480, 640), 4)], ids=lambda v: str(v))
@pytest.mark.parametrize("bigger", [False, True], ids=["same", "one_larger"])
def test_coord_uncaptured_equals_eager_bitwise(api, shape, B, bigger):
    import torch
    preds, gts = _coord_inputs([shape] * B, seed=B + shape[0], bigger=bigger, empty=(1,) if B > 1 else ())
    pred, gt = torch.stack(preds), torch.stack(gts)
    g_ref, g = torch.zeros_like(pred), torch.full_like(pred, 7.0)
    ref, ref_counts = api.coord_loss(pred, gt, CUT, outGradients=g_ref, return_counts=True)
    losses, counts = _coord_async(api, pred, gt, g)
    assert _equal(losses.cpu().numpy(), np.array(ref)) and counts.tolist() == ref_counts
    assert _equal(g.cpu().numpy(), g_ref.cpu().numpy())
    if B > 1:
        assert math.isnan(losses[1].item()) and counts[1].item() == 0
    losses, counts = _coord_async(api, pred, gt, counts=False)
    assert _equal(losses.cpu().numpy(), np.array(ref)) and counts is None


def test_coord_ragged_and_misaligned(api):
    import torch
    shapes = [(60, 80), (7, 5), (45, 61), (30, 3), (480, 640)]
    preds, gts = _coord_inputs(shapes, seed=9, empty=(3,))
    base = torch.empty(3 * 45 * 61 + 1, device="cuda")
    preds[2] = base[1:].view(3, 45, 61).copy_(preds[2])
    grads = [torch.zeros_like(p) for p in preds]
    g_ref = [torch.zeros_like(p) for p in preds]
    ref, ref_counts = api.coord_loss(preds, gts, CUT, outGradients=g_ref, return_counts=True)
    losses, counts = _coord_async(api, preds, gts, grads)
    assert _equal(losses.cpu().numpy(), np.array(ref)) and counts.tolist() == ref_counts
    for a, b in zip(grads, g_ref):
        assert _equal(a.cpu().numpy(), b.cpu().numpy())


def _capture(fn):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def test_reproj_replays_with_new_values_equal_eager(api):
    """One capture, replayed with new predictions, ground truths (every orientation of tests/orientations.py, uniform and
    ill-conditioned ones), pads and cameras copied into its static tensors: bitwise the eager calls on those values."""
    import torch
    B, (H, W), sub = 3, (60, 80), 8
    api.reserve_loss_async(B, H, W)
    pred = torch.zeros(B, 3, H, W, device="cuda")
    gts = torch.zeros(B, 4, 4, device="cuda")
    shifts = torch.zeros(B, 2, dtype=torch.int32, device="cuda")
    cams = torch.zeros(B, 3, device="cuda")
    grads = torch.zeros_like(pred)
    losses = torch.zeros(B, dtype=torch.float64, device="cuda")
    status = torch.zeros(B, dtype=torch.int32, device="cuda")

    def call():
        api.reproj_loss_async(pred, gts, shifts, cams, CUT, sub, losses, status, outGradients=grads, maxReproj=MAXR,
                              minDepth=MIND)

    first = _reproj_inputs([(H, W)] * B, sub, seed=100)
    pred.copy_(torch.stack(first[0])); gts.copy_(first[1]); shifts.copy_(first[2]); cams.copy_(first[3])
    call()                                 # uncaptured warm-up
    g = _capture(call)
    n_rounds = (len(_rotations()) + B - 1) // B + 1
    for k in range(n_rounds):
        p, t, s, c = _reproj_inputs([(H, W)] * B, sub, seed=200 + k, first=k * B)
        pred.copy_(torch.stack(p)); gts.copy_(t); shifts.copy_(s); cams.copy_(c)
        g.replay()
        g_ref = torch.zeros_like(pred)
        ref = _reproj_eager(api, pred, gts, shifts, cams, sub, g_ref)
        assert _equal(losses.cpu().numpy(), np.array(ref)), (k, losses, ref)
        assert status.tolist() == [0] * B
        assert _equal(grads.cpu().numpy(), g_ref.cpu().numpy()), k


def test_coord_replays_with_new_values_equal_eager(api):
    import torch
    B, (H, W) = 2, (60, 80)
    api.reserve_loss_async(B, H + 1, W + 1)
    pred = torch.zeros(B, 3, H + 1, W + 1, device="cuda")
    gt = torch.zeros(B, 3, H, W, device="cuda")
    grads = torch.zeros_like(pred)
    losses = torch.zeros(B, dtype=torch.float64, device="cuda")
    counts = torch.zeros(B, dtype=torch.int64, device="cuda")

    def call():
        api.coord_loss_async(pred, gt, CUT, losses, outGradients=grads, outCounts=counts)

    call()
    g = _capture(call)
    for k in range(4):
        p, q = _coord_inputs([(H, W)] * B, seed=300 + k, bigger=True, empty=(0,) if k == 2 else ())
        pred.copy_(torch.stack(p)); gt.copy_(torch.stack(q))
        g.replay()
        g_ref = torch.zeros_like(pred)
        ref, ref_counts = api.coord_loss(pred, gt, CUT, outGradients=g_ref, return_counts=True)
        assert _equal(losses.cpu().numpy(), np.array(ref)) and counts.tolist() == ref_counts
        assert _equal(grads.cpu().numpy(), g_ref.cpu().numpy())


@pytest.mark.parametrize("singular", ["zero", "nan", "rank2"])
def test_singular_ground_truth_sets_the_status_of_its_image_only(api, singular):
    import torch
    preds, gts, shifts, cams = _reproj_inputs([(60, 80)] * 3, 8, seed=77)
    pred = torch.stack(preds)
    bad = gts.clone()
    if singular == "zero":
        bad[1, :3, :3] = 0.0
    elif singular == "nan":
        bad[1, 0, 0] = float("nan")
    else:
        bad[1, :3, 2] = bad[1, :3, 0]
    with pytest.raises(RuntimeError, match="image 1: ground-truth pose is singular"):
        _reproj_eager(api, pred, bad, shifts, cams, 8, torch.zeros_like(pred))
    g = torch.full_like(pred, 7.0)
    losses, status = _reproj_async(api, pred, bad, shifts, cams, 8, g)
    assert status.tolist() == [0, 1, 0]
    assert math.isnan(losses[1].item())
    assert torch.equal(g[1], torch.zeros_like(g[1]))
    for b in (0, 2):
        g_ref = torch.zeros_like(pred[b:b + 1])
        ref = _reproj_eager(api, pred[b:b + 1], bad[b:b + 1], shifts[b:b + 1], cams[b:b + 1], 8, g_ref)
        assert _equal(losses[b:b + 1].cpu().numpy(), np.array(ref))
        assert _equal(g[b].cpu().numpy(), g_ref[0].cpu().numpy())
    # the same replayed: a graph captured on good values and replayed with the singular one
    gts_s = gts.clone()
    out_l = torch.zeros(3, dtype=torch.float64, device="cuda")
    out_s = torch.zeros(3, dtype=torch.int32, device="cuda")
    api.reserve_loss_async(3, 60, 80)
    graph = _capture(lambda: api.reproj_loss_async(pred, gts_s, shifts, cams, CUT, 8, out_l, out_s, outGradients=g,
                                                   maxReproj=MAXR, minDepth=MIND))
    gts_s.copy_(bad)
    g.fill_(7.0)
    graph.replay()
    assert out_s.tolist() == [0, 1, 0] and math.isnan(out_l[1].item()) and torch.equal(g[1], torch.zeros_like(g[1]))
    assert _equal(out_l[[0, 2]].cpu().numpy(), losses[[0, 2]].cpu().numpy())
    gts_s.copy_(gts)
    graph.replay()
    assert out_s.tolist() == [0, 0, 0] and not math.isnan(out_l[1].item())


def test_no_host_synchronisation(api):
    import torch
    preds, gts, shifts, cams = _reproj_inputs([(60, 80)] * 2, 8, seed=3)
    pred = torch.stack(preds)
    cpreds, cgts = _coord_inputs([(60, 80)] * 2, seed=3)
    cpred, cgt = torch.stack(cpreds), torch.stack(cgts)
    api.reserve_loss_async(2, 60, 80)
    g, cg = torch.zeros_like(pred), torch.zeros_like(cpred)
    losses = torch.zeros(2, dtype=torch.float64, device="cuda")
    status = torch.zeros(2, dtype=torch.int32, device="cuda")
    counts = torch.zeros(2, dtype=torch.int64, device="cuda")
    calls = {"reproj_loss_async": lambda: api.reproj_loss_async(pred, gts, shifts, cams, CUT, 8, losses, status, outGradients=g),
             "coord_loss_async": lambda: api.coord_loss_async(cpred, cgt, CUT, losses, outGradients=cg, outCounts=counts)}
    for fn in calls.values():
        fn()
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    for name, fn in calls.items():
        torch.cuda._sleep(int(2e9))       # ~1 s of device time ahead of the call
        fn()
        assert not stream.query(), f"{name} waited for the device"
        torch.cuda.synchronize()
    # captured in torch's default (global) error mode, with torch work before and after, and replayed
    src = pred.clone()
    doubled = torch.zeros_like(losses)
    for name, fn in calls.items():
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            pred.copy_(src * 1.0)
            fn()
            doubled.copy_(losses * 2.0)
        torch.cuda.synchronize()
        torch.cuda._sleep(int(2e9))
        graph.replay()
        assert not stream.query(), f"the replay of {name} waited for the device"
        torch.cuda.synchronize()
        np.testing.assert_array_equal(doubled.cpu().numpy(), 2.0 * losses.cpu().numpy())


def test_workspace_is_frozen_after_a_capture():
    import torch

    import esac_b200.api as fresh_api
    saved = fresh_api._contexts.get(0)
    ctx = fresh_api.Context(0)        # a context of its own: its workspace has seen only this test
    fresh_api._contexts[0] = ctx
    try:
        preds, gts, shifts, cams = _reproj_inputs([(60, 80)] * 2, 8, seed=4)
        pred = torch.stack(preds)
        losses = torch.zeros(2, dtype=torch.float64, device="cuda")
        status = torch.zeros(2, dtype=torch.int32, device="cuda")
        g = torch.zeros_like(pred)

        def call(p, gg, lo, st, t=gts, s=shifts, c=cams):
            fresh_api.reproj_loss_async(p, t, s, c, CUT, 8, lo, st, outGradients=gg)

        # a first call that is captured cannot create the workspace
        with pytest.raises(RuntimeError, match="reserve_loss_async"):
            _capture(lambda: call(pred, g, losses, status))
        fresh_api.reserve_loss_async(2, 60, 80)
        graph = _capture(lambda: call(pred, g, losses, status))
        graph.replay()
        torch.cuda.synchronize()
        # a larger call fails before enqueuing anything: the outputs are untouched.  The workspace holds per-image records
        # and block partials, not maps, so "larger" takes more images of more blocks each.
        big_p, big_t, big_s, big_c = _reproj_inputs([(240, 320)] * 8, 8, seed=5)
        big = torch.stack(big_p)
        big_g = torch.full_like(big, 7.0)
        big_l = torch.full((8,), -1.0, dtype=torch.float64, device="cuda")
        big_st = torch.full((8,), -1, dtype=torch.int32, device="cuda")
        with pytest.raises(RuntimeError, match="reserve_loss_async"):
            call(big, big_g, big_l, big_st, big_t, big_s, big_c)
        with pytest.raises(RuntimeError, match="reserve_loss_async"):
            fresh_api.reserve_loss_async(8, 240, 320)
        cbig_l = torch.full((8,), -1.0, dtype=torch.float64, device="cuda")
        with pytest.raises(RuntimeError, match="reserve_loss_async"):
            fresh_api.coord_loss_async(big, big, CUT, cbig_l, outGradients=big_g)
        torch.cuda.synchronize()
        assert (big_g == 7.0).all() and (big_l == -1.0).all() and (big_st == -1).all() and (cbig_l == -1.0).all()
        # a smaller call works, and the graph still replays what eager computes
        small = pred[:1, :, :30, :40].contiguous()
        sl = torch.zeros(1, dtype=torch.float64, device="cuda")
        ss = torch.zeros(1, dtype=torch.int32, device="cuda")
        fresh_api.reproj_loss_async(small, gts[:1].contiguous(), shifts[:1].contiguous(), cams[:1].contiguous(), CUT, 8, sl, ss)
        ref = _reproj_eager(fresh_api, small, gts[:1].contiguous(), shifts[:1].contiguous(), cams[:1].contiguous(), 8)
        assert _equal(sl.cpu().numpy(), np.array(ref))
        graph.replay()
        g_ref = torch.zeros_like(pred)
        ref = _reproj_eager(fresh_api, pred, gts, shifts, cams, 8, g_ref)
        assert _equal(losses.cpu().numpy(), np.array(ref)) and _equal(g.cpu().numpy(), g_ref.cpu().numpy())
    finally:
        torch.cuda.synchronize()
        if saved is not None:
            fresh_api._contexts[0] = saved
        else:
            fresh_api._contexts.pop(0, None)
        ctx.close()


class _Net:
    """A stand-in expert: a per-channel affine map of a prior plus a weighted 8x8 average of an image (no convolution,
    whose backward may sum in a different order from one call to the next)."""

    def __init__(self):
        import torch
        self.scale = torch.ones(1, 3, 1, 1, device="cuda", requires_grad=True)
        self.shift = torch.zeros(1, 3, 1, 1, device="cuda", requires_grad=True)
        self.feat = torch.full((1, 3, 1, 1), 0.01, device="cuda", requires_grad=True)

    def parameters(self):
        return [self.scale, self.shift, self.feat]

    def __call__(self, image, prior):
        import torch.nn.functional as F
        return prior * self.scale + self.shift + F.avg_pool2d(image, 8) * self.feat


@pytest.mark.parametrize("loss", ["reproj", "coord"])
def test_captured_training_step_equals_eager_step(api, loss):
    """A stand-in network, the async autograd node, backward() and Adam(capturable=True) in one graph: loss and parameters
    bitwise those of the same steps on the eager node, step by step."""
    import torch

    from esac_b200.autograd import coord_loss, coord_loss_async, reproj_loss, reproj_loss_async
    B, H, W, sub = 2, 60, 80, 8
    image = torch.zeros(B, 1, H * sub, W * sub, device="cuda")
    prior = torch.zeros(B, 3, H, W, device="cuda")
    gts = torch.zeros(B, 4, 4, device="cuda")
    shifts = torch.zeros(B, 2, dtype=torch.int32, device="cuda")
    cams = torch.zeros(B, 3, device="cuda")
    gt_coords = torch.zeros(B, 3, H, W, device="cuda")

    def write(k):
        p, t, s, c = _reproj_inputs([(H, W)] * B, sub, seed=400 + k)
        prior.copy_(torch.stack(p)); gts.copy_(t); shifts.copy_(s); cams.copy_(c)
        image.copy_(torch.rand(image.shape, generator=torch.Generator().manual_seed(k)).cuda())
        gt_coords.copy_(prior + 0.1 * torch.randn(prior.shape, generator=torch.Generator().manual_seed(50 + k)).cuda())
        gt_coords[:, :, ::3, ::2] = 0.0

    def loss_async(pred):
        if loss == "reproj":
            return reproj_loss_async(pred, gts, shifts, cams, CUT, sub)
        return coord_loss_async(pred, gt_coords, CUT)

    def loss_eager(pred):
        if loss == "reproj":
            s, c = shifts.cpu().numpy(), cams.cpu().numpy()
            return reproj_loss(pred, gts, c[:, 0], s[:, 0], s[:, 1], CUT, sub, c[:, 1], c[:, 2])
        return coord_loss(pred, gt_coords, CUT)

    net, ref = _Net(), _Net()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3, capturable=True)
    opt_ref = torch.optim.Adam(ref.parameters(), lr=1e-3, capturable=True)
    api.reserve_loss_async(B, H, W)
    write(0)

    def step():
        opt.zero_grad(set_to_none=False)
        out = loss_async(net(image, prior))
        out.backward()
        opt.step()
        return out

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up outside the capture (Adam's state, cuDNN), mirrored on the reference
        for _ in range(2):
            step()
            opt_ref.zero_grad(set_to_none=False)
            loss_eager(ref(image, prior)).backward()
            opt_ref.step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for k in range(1, 5):
        write(k)
        graph.replay()
        opt_ref.zero_grad(set_to_none=False)
        want = loss_eager(ref(image, prior))
        want.backward()
        opt_ref.step()
        assert _equal(out.detach().cpu().numpy(), want.detach().cpu().numpy()), (k, out.item(), want.item())
        for a, b in zip(net.parameters(), ref.parameters()):
            assert torch.equal(a, b), k


@pytest.mark.parametrize("example", ["init_expert_step_graph_synthetic.py", "ref_expert_step_graph_synthetic.py"])
def test_graph_examples_check_against_the_eager_steps(example):
    import runpy
    import sys
    from pathlib import Path
    ex = Path(__file__).resolve().parents[1] / "examples" / example
    argv = sys.argv
    sys.argv = [str(ex), "--iterations", "4", "--check"]
    try:
        mod = runpy.run_path(str(ex), run_name="example")
        assert mod["main"]() == 0
    finally:
        sys.argv = argv
