"""GPU tests of the batched entry points with a camera per image (forward_batch, backward_batch, reproj_loss,
autograd.esac_loss_batch): a batch whose images each carry their own shift, focal length and principal point must give
what a loop of single-image calls with those cameras gives, and one camera broadcast to every image must give bitwise
what the scalar call gives."""
import copy

import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error

pytestmark = pytest.mark.gpu

# four cameras of a mixed dataset (7Scenes' 525 among calibrated ones), principal points off the image centre
F = [450.0, 525.0, 572.3, 700.0]
PPX = [171.7, 150.0, 145.5, 168.25]    # 30x40 maps at sub 8: the image is 320 x 240
PPY = [110.2, 131.0, 120.0, 105.5]
SX = [-4, 3, 0, 2]
SY = [2, -3, 4, -1]


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 0)
    return api


def _scenes(E, H, W, M, seed):
    return [make_scene(E=E, H=H, W=W, M=M, sub=8, seed=seed + b, f=F[b], ppx=PPX[b], ppy=PPY[b], shiftX=SX[b], shiftY=SY[b])
            for b in range(len(F))]


def _cameras(kind):
    """The five per-image arguments as a DataLoader-like caller may hold them."""
    import torch
    vals = (SX, SY, F, PPX, PPY)
    if kind == "numpy":
        return tuple(np.array(v) for v in vals)
    dev = "cuda" if kind == "cuda" else "cpu"
    return (torch.tensor(SX, device=dev), torch.tensor(SY, device=dev), torch.tensor(F, dtype=torch.float64, device=dev),
            torch.tensor(PPX, dtype=torch.float64, device=dev), torch.tensor(PPY, dtype=torch.float64, device=dev))


@pytest.mark.parametrize("kind", ["numpy", "cpu", "cuda"])
def test_forward_batch_with_a_camera_per_image_equals_a_loop_of_forward(api, kind):
    import torch
    scenes = _scenes(3, 30, 40, 48, 70)
    B = len(scenes)
    coords = np.stack([s.coords for s in scenes])
    assign = np.stack([s.assign for s in scenes])
    tail = scenes[0].params[5:]   # tau, alpha, beta, maxReproj, sub: one value per run
    api.set_seed(321)
    ref_e, ref_p = [], []
    for s in scenes:
        out = np.zeros((4, 4), np.float32)
        ref_e.append(api.forward(s.coords, s.assign, out, *s.params))
        ref_p.append(out)
    ref_p = np.stack(ref_p)
    api.set_seed(321)
    if kind == "numpy":
        outs = np.zeros((B, 4, 4), np.float32)
        e = api.forward_batch(coords, assign, outs, *_cameras(kind), *tail)
    else:
        dev = "cuda" if kind == "cuda" else "cpu"
        t_outs = torch.zeros(B, 4, 4, device=dev)
        e = api.forward_batch(torch.from_numpy(coords).to(dev), torch.from_numpy(assign).to(dev), t_outs, *_cameras(kind), *tail)
        outs = t_outs.cpu().numpy()
    assert e == ref_e == [s.gt_expert for s in scenes]
    assert np.array_equal(outs, ref_p)
    for b, s in enumerate(scenes):
        rot, trans = pose_error(outs[b], s.gt_pose)
        assert rot < 1.0 and trans < 0.05, (b, rot, trans)


def test_forward_batch_with_swapped_cameras_misses_the_ground_truth(api):
    """The maps were generated through their own cameras: handing image b the camera of image b+1 must show."""
    scenes = _scenes(3, 30, 40, 48, 70)
    coords = np.stack([s.coords for s in scenes])
    assign = np.stack([s.assign for s in scenes])
    roll = [np.roll(np.array(v), 1) for v in (SX, SY, F, PPX, PPY)]
    outs = np.zeros((len(scenes), 4, 4), np.float32)
    api.forward_batch(coords, assign, outs, *roll, *scenes[0].params[5:])
    errs = [pose_error(outs[b], s.gt_pose) for b, s in enumerate(scenes)]
    assert all(rot >= 1.0 or trans >= 0.05 for rot, trans in errs), errs


@pytest.mark.parametrize("workers", [1, 4])
@pytest.mark.parametrize("kind", ["cpu", "cuda"])
def test_backward_batch_with_a_camera_per_image_equals_a_loop_of_backward(api, workers, kind):
    import torch
    scenes = _scenes(3, 24, 32, 24, 40)
    B = len(scenes)
    coords = np.stack([s.coords for s in scenes])
    assign = np.stack([s.assign for s in scenes])
    gts = np.stack([s.gt_pose for s in scenes])
    tail = scenes[0].params[5:]
    ctx = api.context()
    ctx.set_option("batch_workers", workers)
    try:
        api.set_seed(19)
        g_loop = np.zeros_like(coords)
        l_loop = [api.backward(s.coords, g_loop[b], s.assign, s.gt_pose, 1.0, 100.0, 100.0, *s.params)
                  for b, s in enumerate(scenes)]
        api.set_seed(19)
        dev = "cuda" if kind == "cuda" else "cpu"
        t_grads = torch.zeros(coords.shape, device=dev)
        losses = api.backward_batch(torch.from_numpy(coords).to(dev), t_grads, torch.from_numpy(assign).to(dev),
                                    torch.from_numpy(gts).to(dev), 1.0, 100.0, 100.0, *_cameras(kind), *tail)
    finally:
        ctx.set_option("batch_workers", 8)
    assert np.allclose(losses, l_loop, rtol=1e-12, atol=0)
    assert np.array_equal(t_grads.cpu().numpy(), g_loop)


def test_one_camera_broadcast_to_every_image_equals_the_scalar_call(api):
    scenes = [make_scene(E=3, H=24, W=32, M=24, sub=8, seed=80 + b) for b in range(3)]
    B = len(scenes)
    coords = np.stack([s.coords for s in scenes])
    assign = np.stack([s.assign for s in scenes])
    gts = np.stack([s.gt_pose for s in scenes])
    sx, sy, f, ppx, ppy = 2, -1, 571.9, 131.3, 97.6
    tail = scenes[0].params[5:]
    arrays = (np.full(B, sx), np.full(B, sy), np.full(B, f), np.full(B, ppx), np.full(B, ppy))
    # forward_batch
    res = []
    for cam in ((sx, sy, f, ppx, ppy), arrays):
        api.set_seed(5)
        outs = np.zeros((B, 4, 4), np.float32)
        res.append((api.forward_batch(coords, assign, outs, *cam, *tail), outs))
    assert res[0][0] == res[1][0] and np.array_equal(res[0][1], res[1][1])
    # backward_batch
    res = []
    for cam in ((sx, sy, f, ppx, ppy), arrays):
        api.set_seed(6)
        g = np.zeros_like(coords)
        res.append((api.backward_batch(coords, g, assign, gts, 1.0, 100.0, 100.0, *cam, *tail), g))
    assert res[0][0] == res[1][0] and np.array_equal(res[0][1], res[1][1])
    # reproj_loss
    _, pred, gts = _reproj_case(24, 32, 700)
    arrays = tuple(np.full(len(pred), v) for v in (sx, sy, f, ppx, ppy))
    res = []
    for cam in ((sx, sy, f, ppx, ppy), arrays):
        g = np.zeros_like(pred)
        res.append((api.reproj_loss(pred, gts, cam[2], cam[0], cam[1], 10.0, 8, cam[3], cam[4], outGradients=g), g))
    assert res[0][0] == res[1][0] and np.array_equal(res[0][1], res[1][1])


def _reproj_case(H, W, seed):
    scenes = [make_scene(E=1, H=H, W=W, M=8, sub=8, seed=seed + b, f=F[b], ppx=PPX[b] * W / 40, ppy=PPY[b] * H / 30,
                         shiftX=SX[b], shiftY=SY[b]) for b in range(len(F))]
    pred = np.stack([s.coords[0] for s in scenes])
    gts = np.stack([s.gt_pose for s in scenes])
    return scenes, pred, gts


@pytest.mark.parametrize("H,W", [(60, 80), (33, 47)])   # the sizes of test_gpu_reproj.py; 33x47: the scalar load path
@pytest.mark.parametrize("kind", ["cpu", "cuda"])
def test_reproj_loss_with_a_camera_per_image(kind, H, W):
    import torch
    import esac_b200.api as api
    from oracle.reproj_loss_oracle import reproj_errors, reproj_loss_and_grad
    scenes, pred, gts = _reproj_case(H, W, 500 + H)
    pred[0, :, 0, 0] = [0.0, 0.0, -50.0]       # behind the camera -> depth clamp
    pred[1, :, 1, 1] = [1e4, -1e4, 3.0]        # error far beyond 100 px -> zero gradient
    B, cut = len(scenes), 10.0
    f = torch.tensor([s.f for s in scenes], dtype=torch.float64)
    cx = [s.ppx for s in scenes]
    cy = np.array([s.ppy for s in scenes])
    dev = "cuda" if kind == "cuda" else "cpu"
    tp = torch.from_numpy(pred).to(dev)
    tg = torch.full(pred.shape, 7.0, device=dev)      # overwritten, not accumulated
    losses = api.reproj_loss(tp, torch.from_numpy(gts).to(dev), f.to(dev), SX, SY, cut, 8, cx, cy, outGradients=tg)
    g = tg.cpu().numpy()
    for b, s in enumerate(scenes):
        # one image, one camera
        g1 = np.zeros_like(pred[b:b + 1])
        l1 = api.reproj_loss(pred[b:b + 1], gts[b:b + 1], s.f, SX[b], SY[b], cut, 8, s.ppx, s.ppy, outGradients=g1)
        assert np.array_equal(g[b], g1[0]), b
        assert abs(losses[b] - l1[0]) <= 1e-12 * abs(l1[0]), (b, losses[b], l1[0])
        # the float64 yardstick, at the bar of test_gpu_reproj.py
        iw, ih = 2 * s.ppx, 2 * s.ppy
        _, g32 = reproj_loss_and_grad(pred[b], gts[b], s.f, SX[b], SY[b], cut, 8, iw, ih)
        l64, g64 = reproj_loss_and_grad(pred[b], gts[b], s.f, SX[b], SY[b], cut, 8, iw, ih, dtype=torch.float64)
        assert abs(losses[b] - l64) <= 1e-5 * max(1.0, abs(l64)), (b, losses[b], l64)
        e64 = reproj_errors(torch.from_numpy(pred[b]), torch.from_numpy(gts[b]), s.f, SX[b], SY[b], 8, iw, ih,
                            dtype=torch.float64).numpy().reshape(H, W)
        kink = (np.abs(e64 - cut) < 1e-3) | (np.abs(e64 - 100.0) < 1e-3) & (e64 < 100.0)
        assert kink.sum() <= 2e-4 * H * W + 2
        keep = ~kink[None]
        d32 = (g32.double() - g64).numpy() * keep
        dk = (g[b] - g64.numpy()) * keep
        scale = g64.abs().max().item()
        assert np.sqrt((dk ** 2).mean()) <= 1.5 * np.sqrt((d32 ** 2).mean()) + 1e-7 * scale
        assert np.abs(dk).max() <= 4 * np.abs(d32).max() + 1e-6 * scale


def test_reproj_loss_autograd_node_takes_a_camera_per_image():
    import torch
    from esac_b200.autograd import reproj_loss
    scenes, pred, gts = _reproj_case(24, 32, 900)
    f = torch.tensor([s.f for s in scenes], dtype=torch.float64)
    cx, cy = [s.ppx for s in scenes], [s.ppy for s in scenes]
    p = torch.from_numpy(pred).cuda().requires_grad_(True)
    loss = reproj_loss(p, torch.from_numpy(gts).cuda(), f, SX, SY, 10.0, 8, cx, cy)
    (loss * 3.0).backward()
    ref, ref_g = 0.0, []
    for b, s in enumerate(scenes):
        q = torch.from_numpy(pred[b:b + 1]).cuda().requires_grad_(True)
        lb = reproj_loss(q, torch.from_numpy(gts[b:b + 1]).cuda(), s.f, SX[b], SY[b], 10.0, 8, s.ppx, s.ppy)
        (lb * 3.0 / len(scenes)).backward()
        ref += lb.item() / len(scenes)
        ref_g.append(q.grad[0])
    assert abs(loss.item() - ref) <= 1e-6 * abs(ref)
    assert torch.allclose(p.grad, torch.stack(ref_g), rtol=1e-6, atol=0)


def _loss_batch_inputs(expert_selection):
    import torch
    scenes = _scenes(3, 24, 32, 24, 40)
    coords = torch.from_numpy(np.stack([s.coords for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    if expert_selection:
        assign = torch.tensor([s.gt_expert for s in scenes], device="cuda")[:, None].expand(len(scenes), 24)
    else:
        assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    params = (1.0, 100.0, 100.0) + _cameras("cpu") + scenes[0].params[5:]
    per_image = [(1.0, 100.0, 100.0) + s.params for s in scenes]
    return scenes, coords, assign, gts, params, per_image


@pytest.mark.parametrize("expert_selection", [False, True])
def test_esac_loss_batch_gradients(api, expert_selection):
    import torch
    from esac_b200.autograd import esac_loss, esac_loss_batch
    scenes, coords, assign, gts, params, per_image = _loss_batch_inputs(expert_selection)
    B, E = coords.shape[:2]
    logits = torch.randn(B, E, generator=torch.Generator().manual_seed(3)).cuda()
    # batched node
    api.set_seed(41)
    c = coords.clone().requires_grad_(True)
    lp = torch.log_softmax(logits, 1).detach().requires_grad_(True)
    losses = esac_loss_batch(c, lp, assign, gts, *params)
    assert losses.shape == (B,)
    losses.sum().backward()
    # its coordinate gradient is backward_batch's
    api.set_seed(41)
    g_ref = torch.zeros_like(coords)
    l_ref = api.backward_batch(coords, g_ref, assign, gts, *params)
    assert losses.tolist() == torch.tensor(l_ref, dtype=torch.float32).tolist()
    assert torch.equal(c.grad, g_ref)
    # its gating gradient is that of B esac_loss calls
    api.set_seed(41)
    lp1 = lp.detach().clone().requires_grad_(True)
    total = sum(esac_loss(coords[b], lp1[b], assign[b], gts[b], *per_image[b]) for b in range(B))
    total.backward()
    assert torch.allclose(lp.grad, lp1.grad, rtol=1e-6, atol=0)
    if expert_selection:
        nz = lp.grad.cpu().numpy() != 0
        assert (nz.sum(1) == 1).all() and [int(np.flatnonzero(r)[0]) for r in nz] == [s.gt_expert for s in scenes]


def test_esac_loss_batch_optimiser_step_equals_the_per_image_loop(api):
    """One training step on stand-in networks (a learnable affine map of each expert's coordinate prior, a linear gating
    head; cf. examples/train_step_synthetic.py) through esac_loss_batch and through B esac_loss calls: same parameters."""
    import torch
    import torch.nn as nn
    from esac_b200.autograd import esac_loss, esac_loss_batch
    scenes, coords, assign, gts, params, per_image = _loss_batch_inputs(False)
    B, E = coords.shape[:2]

    class Nets(nn.Module):
        def __init__(self):
            super().__init__()
            self.scale = nn.Parameter(torch.ones(E, 3, 1, 1))
            self.shift = nn.Parameter(torch.zeros(E, 3, 1, 1))
            self.gating = nn.Linear(16, E)

        def forward(self, prior, feats):
            return prior * self.scale + self.shift, torch.log_softmax(self.gating(feats), 1)

    torch.manual_seed(0)
    nets = Nets().cuda()
    feats = torch.randn(B, 16, generator=torch.Generator().manual_seed(1)).cuda()
    prior = coords + 0.01 * torch.randn(coords.shape, generator=torch.Generator().manual_seed(2)).cuda()
    after = []
    for batched in (True, False):
        m = copy.deepcopy(nets)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        opt.zero_grad()
        pred, lp = m(prior, feats)
        api.set_seed(77)
        if batched:
            esac_loss_batch(pred, lp, assign, gts, *params).sum().backward()
        else:
            sum(esac_loss(pred[b], lp[b], assign[b], gts[b], *per_image[b]) for b in range(B)).backward()
        opt.step()
        after.append([p.detach().cpu().numpy() for p in m.parameters()])
    for a, b, p0 in zip(after[0], after[1], nets.parameters()):
        assert np.array_equal(a, b)
        assert not np.array_equal(a, p0.detach().cpu().numpy())   # the step did move every parameter
