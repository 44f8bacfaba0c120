"""GPU tests of ragged batches: the batched entry points on a list of per-image tensors, each image with its own map size
(19Scenes, Aachen and Dubrovnik keep each image's aspect ratio).  Image b must compute what a single-image call on it
computes -- the same poses and experts, the same minimal sets, bitwise the same losses and gradients -- and a list of
equal-shaped tensors must give bitwise what the stacked tensor gives."""
import copy
import ctypes as C

import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error
from test_gpu_coord_loss import _case as _coord_case, _check_against_oracle as _coord_oracle_bar

pytestmark = pytest.mark.gpu

# portrait and landscape; N = 1200 and 972 (N % 4 == 0: 128-bit / TMA-style scoring loads), 1395 and 1147 (odd N: scalar)
SHAPES = [(30, 40), (40, 30), (31, 45), (37, 31)]
F = [450.0, 525.0, 572.3, 700.0]
SX = [-4, 3, 0, 2]
SY = [2, -3, 4, -1]
TAIL = (10.0, 100.0, 0.5, 100.0, 8)


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 0)
    return api


def _scenes(E, M, seed, shapes=SHAPES):
    out = []
    for b, (h, w) in enumerate(shapes):
        out.append(make_scene(E=E, H=h, W=w, M=M, sub=8, seed=seed + b, f=F[b % 4], ppx=w * 4 + 3.5 * b, ppy=h * 4 - 2.25 * b,
                              shiftX=SX[b % 4], shiftY=SY[b % 4]))
    return out


def _cams(scenes):
    return ([s.shiftX for s in scenes], [s.shiftY for s in scenes], [s.f for s in scenes], [s.ppx for s in scenes],
            [s.ppy for s in scenes])


def _to(arrays, kind):
    import torch
    if kind == "numpy":
        return list(arrays)
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda" if kind == "cuda" else "cpu") for a in arrays]


# ---- forward / backward -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["cpu", "cuda"])
def test_forward_list_equals_a_loop_of_forward(api, kind):
    import torch
    scenes = _scenes(3, 48, 70)
    B = len(scenes)
    api.set_seed(321)
    ref_e, ref_p = [], []
    for s in scenes:
        out = np.zeros((4, 4), np.float32)
        ref_e.append(api.forward(s.coords, s.assign, out, *s.params))
        ref_p.append(out)
    api.set_seed(321)
    dev = "cuda" if kind == "cuda" else "cpu"
    outs = torch.zeros(B, 4, 4, device=dev)
    e = api.forward_batch(_to([s.coords for s in scenes], kind), torch.from_numpy(np.stack([s.assign for s in scenes])).to(dev),
                          outs, *_cams(scenes), *TAIL)
    outs = outs.cpu().numpy()
    assert e == ref_e == [s.gt_expert for s in scenes]
    assert np.array_equal(outs, np.stack(ref_p))
    for b, s in enumerate(scenes):
        rot, trans = pose_error(outs[b], s.gt_pose)
        assert rot < 1.0 and trans < 0.05, (b, rot, trans)


@pytest.mark.parametrize("workers", [1, 8])
@pytest.mark.parametrize("kind", ["cpu", "cuda"])
def test_backward_list_equals_a_loop_of_backward(api, workers, kind):
    import torch
    scenes = _scenes(3, 24, 40)
    B = len(scenes)
    gts = np.stack([s.gt_pose for s in scenes])
    ctx = api.context()
    ctx.set_option("batch_workers", workers)
    try:
        api.set_seed(19)
        g_loop = [np.zeros_like(s.coords) for s in scenes]
        l_loop = [api.backward(s.coords, g_loop[b], s.assign, s.gt_pose, 1.0, 100.0, 100.0, *s.params)
                  for b, s in enumerate(scenes)]
        api.set_seed(19)
        dev = "cuda" if kind == "cuda" else "cpu"
        grads = [torch.zeros(s.coords.shape, device=dev) for s in scenes]
        losses = api.backward_batch(_to([s.coords for s in scenes], kind), grads,
                                    torch.from_numpy(np.stack([s.assign for s in scenes])).to(dev), torch.from_numpy(gts).to(dev),
                                    1.0, 100.0, 100.0, *_cams(scenes), *TAIL)
    finally:
        ctx.set_option("batch_workers", 8)
    assert np.allclose(losses, l_loop, rtol=1e-12, atol=0)
    for b in range(B):
        assert np.array_equal(grads[b].cpu().numpy(), g_loop[b]), b


# ---- loss kernels -------------------------------------------------------------------------------------------------
def _misaligned(a):
    """A contiguous CUDA copy of `a` whose storage starts 4 bytes past a 16-byte boundary: the scalar load path."""
    import torch
    flat = torch.empty(a.size + 1, device="cuda")
    v = flat[1:].view(a.shape)
    v.copy_(torch.from_numpy(a))
    assert v.data_ptr() % 16 == 4 and v.is_contiguous()
    return v


# (H, W): vector path, odd W with N % 4 == 0 (vector path), odd N (scalar), portrait; "mis" = misaligned storage
REPROJ = [(24, 32, ""), (36, 31, ""), (33, 47, ""), (40, 30, "mis"), (29, 35, "")]


def _reproj_inputs(seed):
    scenes = [make_scene(E=1, H=h, W=w, M=8, sub=8, seed=seed + b, f=F[b % 4], shiftX=SX[b % 4], shiftY=SY[b % 4])
              for b, (h, w, _) in enumerate(REPROJ)]
    preds = [s.coords[0] for s in scenes]
    preds[0][:, 0, 0] = [0.0, 0.0, -50.0]       # behind the camera -> depth clamp
    preds[1][:, 1, 1] = [1e4, -1e4, 3.0]        # error far beyond 100 px -> zero gradient
    return scenes, preds, np.stack([s.gt_pose for s in scenes])


def _device_list(arrays, layout, kind):
    import torch
    if kind == "cpu":
        return [torch.from_numpy(np.ascontiguousarray(a)) for a in arrays]
    return [_misaligned(a) if m == "mis" else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a, m in zip(arrays, layout)]


@pytest.mark.parametrize("order", ["vector_first", "scalar_first"])
@pytest.mark.parametrize("grad", [True, False])
@pytest.mark.parametrize("kind", ["cpu", "cuda"])
def test_reproj_loss_list_is_bitwise_per_image(api, kind, grad, order):
    import torch
    from oracle.reproj_loss_oracle import reproj_errors, reproj_loss_and_grad
    scenes, preds, gts = _reproj_inputs(600)
    layout = [m for _, _, m in REPROJ]
    f = F[:4] + F[:1]
    sx, sy = [SX[b % 4] for b in range(len(REPROJ))], [SY[b % 4] for b in range(len(REPROJ))]
    if order == "scalar_first":   # image 0 on the scalar path, later images on the 128-bit one
        scenes, preds, gts, layout, f, sx, sy = (v[::-1] for v in (scenes, preds, gts, layout, f, sx, sy))
        gts = np.ascontiguousarray(gts)
    f = torch.tensor(f, dtype=torch.float64)
    cut = 10.0
    pr = _device_list(preds, layout, kind)
    og = [torch.full_like(p, 7.0) for p in pr] if grad else None     # overwritten, not accumulated
    losses = api.reproj_loss(pr, torch.from_numpy(gts), f, sx, sy, cut, 8, outGradients=og)
    for b, s in enumerate(scenes):
        H, W = preds[b].shape[1:]
        one = pr[b][None]                        # the same storage: the same load path as in the list
        g1 = torch.empty_like(one) if grad else None
        l1 = api.reproj_loss(one, torch.from_numpy(gts[b:b + 1]), float(f[b]), sx[b], sy[b], cut, 8, outGradients=g1)
        assert losses[b] == l1[0], (b, losses[b], l1[0])
        if grad:
            assert torch.equal(og[b].cpu(), g1[0].cpu()), b
        # the float64 yardstick at the bar of test_gpu_reproj.py
        l64, g64 = reproj_loss_and_grad(preds[b], gts[b], float(f[b]), sx[b], sy[b], cut, 8, dtype=torch.float64)
        assert abs(losses[b] - l64) <= 1e-5 * max(1.0, abs(l64)), (b, losses[b], l64)
        if grad:
            _, g32 = reproj_loss_and_grad(preds[b], gts[b], float(f[b]), sx[b], sy[b], cut, 8)
            e64 = reproj_errors(torch.from_numpy(preds[b]), torch.from_numpy(gts[b]), float(f[b]), sx[b], sy[b], 8,
                                dtype=torch.float64).numpy().reshape(H, W)
            kink = (np.abs(e64 - cut) < 1e-3) | (np.abs(e64 - 100.0) < 1e-3) & (e64 < 100.0)
            assert kink.sum() <= 2e-4 * H * W + 2
            keep = ~kink[None]
            d32 = (g32.double() - g64).numpy() * keep
            dk = (og[b].cpu().double().numpy() - g64.numpy()) * keep
            scale = g64.abs().max().item()
            assert np.sqrt((dk ** 2).mean()) <= 1.5 * np.sqrt((d32 ** 2).mean()) + 1e-7 * scale, b
            assert np.abs(dk).max() <= 4 * np.abs(d32).max() + 1e-6 * scale, b
    if not grad:
        assert all(np.isfinite(losses))


def test_reproj_loss_list_default_principal_point_is_per_image(api):
    scenes, preds, gts = _reproj_inputs(640)
    losses = api.reproj_loss(preds, gts, 525.0, 0, 0, 10.0, 8)
    for b, p in enumerate(preds):
        H, W = p.shape[1:]
        assert losses[b] == api.reproj_loss(p[None], gts[b:b + 1], 525.0, 0, 0, 10.0, 8, W * 4.0, H * 4.0)[0], b


# (Hp, Wp, Hg, Wg): equal sizes on the vector path, crops in both directions, odd sizes, misaligned storage
COORD = [(24, 32, 24, 32, ""), (25, 33, 24, 32, ""), (30, 40, 31, 41, ""), (33, 47, 33, 47, ""), (24, 32, 25, 32, ""),
         (32, 24, 32, 24, "mis")]


@pytest.mark.parametrize("grad", [True, False])
@pytest.mark.parametrize("kind", ["cpu", "cuda"])
def test_coord_loss_list_is_bitwise_per_image(api, kind, grad):
    import torch
    preds, gts = [], []
    for i, (hp, wp, hg, wg, _) in enumerate(COORD):
        p, g = _coord_case(1, hp, wp, seed=300 + i, Hg=hg, Wg=wg, invalid=0.3)
        preds.append(p[0])
        gts.append(g[0])
    gts[3][:] = 0.0                            # an image without a valid cell: NaN loss, zero gradient
    layout = [m for *_, m in COORD]
    pr, gt = _device_list(preds, layout, kind), _device_list(gts, layout, kind)
    og = [torch.full_like(p, 7.0) for p in pr] if grad else None
    losses, counts = api.coord_loss(pr, gt, 100.0, outGradients=og, return_counts=True)
    for b in range(len(COORD)):
        g1 = torch.empty_like(pr[b][None]) if grad else None
        l1, c1 = api.coord_loss(pr[b][None], gt[b][None], 100.0, outGradients=g1, return_counts=True)
        assert counts[b] == c1[0]
        assert np.array_equal(np.float64(losses[b]), np.float64(l1[0]), equal_nan=True), (b, losses[b], l1[0])
        if grad:
            assert torch.equal(og[b].cpu(), g1[0].cpu()), b
    assert np.isnan(losses[3]) and counts[3] == 0
    if grad:
        assert (og[3] == 0).all()
        for b in range(len(COORD)):
            if b != 3:   # the float64-oracle bar of test_gpu_coord_loss.py, image by image
                _coord_oracle_bar(preds[b][None], gts[b][None], [losses[b]], [counts[b]], og[b].cpu().numpy()[None])


# ---- uniform lists, stream ordering, the C ABI ------------------------------------------------------------------
def test_a_list_of_equal_shapes_is_bitwise_the_stacked_call(api):
    import torch
    scenes = [make_scene(E=3, H=24, W=32, M=24, sub=8, seed=80 + b, f=F[b]) for b in range(3)]
    coords = np.stack([s.coords for s in scenes])
    assign = np.stack([s.assign for s in scenes])
    gts = np.stack([s.gt_pose for s in scenes])
    cams = _cams(scenes)
    res = []
    for c in (coords, list(coords)):
        api.set_seed(5)
        outs = np.zeros((3, 4, 4), np.float32)
        res.append((api.forward_batch(c, assign, outs, *cams, *TAIL), outs))
    assert res[0][0] == res[1][0] and np.array_equal(res[0][1], res[1][1])
    res = []
    for listed in (False, True):
        api.set_seed(6)
        g = np.zeros_like(coords)
        c, gg = (list(coords), list(g)) if listed else (coords, g)
        res.append((api.backward_batch(c, gg, assign, gts, 1.0, 100.0, 100.0, *cams, *TAIL), g))
    assert res[0][0] == res[1][0] and np.array_equal(res[0][1], res[1][1])
    pred = torch.from_numpy(coords[:, 0].copy()).cuda()
    tg = torch.from_numpy(gts).cuda()
    for H, W in ((24, 32), (23, 31)):
        p = pred[:, :, :H, :W].contiguous()
        ga, gb = torch.empty_like(p), torch.empty_like(p)
        la = api.reproj_loss(p, tg, cams[2], 0, 0, 10.0, 8, outGradients=ga)
        lb = api.reproj_loss(list(p.unbind(0)), tg, cams[2], 0, 0, 10.0, 8, outGradients=list(gb.unbind(0)))
        assert la == lb and torch.equal(ga, gb)
        q = (p + 0.5 * torch.randn_like(p)).contiguous()
        la, ca = api.coord_loss(p, q, 1.0, outGradients=ga, return_counts=True)
        lb, cb = api.coord_loss(list(p.unbind(0)), list(q.unbind(0)), 1.0, outGradients=list(gb.unbind(0)), return_counts=True)
        assert la == lb and ca == cb and torch.equal(ga, gb)


def test_cuda_lists_run_on_the_current_stream(api):
    import torch
    _, preds, gts = _reproj_inputs(700)
    side = torch.cuda.Stream()
    ref = api.reproj_loss(preds, gts, 525.0, 0, 0, 10.0, 8)
    with torch.cuda.stream(side):
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(4):
            big = big @ big / 64.0                    # keep the side stream busy
        pr = [torch.from_numpy(p).cuda() * 1.0 for p in preds]   # produced on the side stream
        og = [torch.empty_like(p) for p in pr]
        losses = api.reproj_loss(pr, torch.from_numpy(gts).cuda(), 525.0, 0, 0, 10.0, 8, outGradients=og)
        doubled = [g * 2.0 for g in og]                # consumes the gradients on the same stream
    torch.cuda.synchronize()
    assert losses == ref
    g_ref = [np.zeros_like(p) for p in preds]
    api.reproj_loss(preds, gts, 525.0, 0, 0, 10.0, 8, outGradients=g_ref)
    for d, g in zip(doubled, g_ref):
        assert np.array_equal(d.cpu().numpy(), 2.0 * g)


def test_host_and_device_pointers_mixed_in_one_argument_are_rejected(api):
    import torch
    ctx = api.context()
    ctx.set_stream(0)
    _, preds, gts = _reproj_inputs(720)
    p_dev = torch.from_numpy(preds[0]).cuda()
    p_host = np.ascontiguousarray(preds[1])
    ptrs = (C.c_void_p * 2)(p_dev.data_ptr(), p_host.ctypes.data)
    hs = np.array([p.shape[1] for p in preds[:2]], np.int32)
    ws = np.array([p.shape[2] for p in preds[:2]], np.int32)
    cam = [np.array(v, np.float32) for v in ([525.0, 525.0], [100.0, 100.0], [80.0, 80.0])]
    losses = np.zeros(2)
    g = np.ascontiguousarray(gts[:2])
    rc = ctx.lib.esacb200_reproj_loss_ragged(ctx.handle, 2, ptrs, None, hs.ctypes.data, ws.ctypes.data, g.ctypes.data, None, None,
                                             cam[0].ctypes.data, cam[1].ctypes.data, cam[2].ctypes.data, 8, 10.0, 100.0, 0.1,
                                             losses.ctypes.data)
    assert rc < 0 and b"mixes host and device pointers" in ctx.lib.esacb200_last_error(ctx.handle)
    counts = np.zeros(2, np.int64)
    rc = ctx.lib.esacb200_coord_loss_ragged(ctx.handle, 2, ptrs, hs.ctypes.data, ws.ctypes.data, ptrs, hs.ctypes.data, ws.ctypes.data,
                                            None, 100.0, losses.ctypes.data, counts.ctypes.data)
    assert rc < 0 and b"mixes host and device pointers" in ctx.lib.esacb200_last_error(ctx.handle)
    # per-image size errors name the image
    bad = np.array([p.shape[1] for p in preds[:2]], np.int32)
    bad[1] += 2
    rc = ctx.lib.esacb200_coord_loss_ragged(ctx.handle, 2, ptrs, hs.ctypes.data, ws.ctypes.data, ptrs, bad.ctypes.data, ws.ctypes.data,
                                            None, 100.0, losses.ctypes.data, counts.ctypes.data)
    assert rc < 0 and b"image 1: size mismatch" in ctx.lib.esacb200_last_error(ctx.handle)
    # the forward and backward entry points check every argument the same way
    scenes = _scenes(2, 8, 90, shapes=SHAPES[:2])
    c_dev = torch.from_numpy(scenes[0].coords).cuda()
    cptrs = (C.c_void_p * 2)(c_dev.data_ptr(), scenes[1].coords.ctypes.data)
    hs2 = np.array([s.coords.shape[2] for s in scenes], np.int32)
    ws2 = np.array([s.coords.shape[3] for s in scenes], np.int32)
    assign = np.ascontiguousarray(np.stack([s.assign for s in scenes]))
    outs = np.zeros((2, 4, 4), np.float32)
    c2 = [np.array(v, np.float32) for v in _cams(scenes)[2:]]
    rc = ctx.lib.esacb200_forward_ragged(ctx.handle, 2, cptrs, hs2.ctypes.data, ws2.ctypes.data, 2, assign.ctypes.data, 1, 8,
                                         outs.ctypes.data, None, None, c2[0].ctypes.data, c2[1].ctypes.data, c2[2].ctypes.data,
                                         *TAIL, None)
    assert rc < 0 and b"mixes host and device pointers" in ctx.lib.esacb200_last_error(ctx.handle)


# ---- autograd ---------------------------------------------------------------------------------------------------
def test_esac_loss_batch_on_a_list_optimiser_step_equals_the_per_image_loop(api):
    import torch
    import torch.nn as nn
    from esac_b200.autograd import esac_loss, esac_loss_batch
    scenes = _scenes(3, 24, 40)
    B, E = len(scenes), 3
    coords = [torch.from_numpy(s.coords).cuda() for s in scenes]
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    params = (1.0, 100.0, 100.0) + _cams(scenes) + TAIL
    per_image = [(1.0, 100.0, 100.0) + s.params for s in scenes]

    class Nets(nn.Module):
        def __init__(self):
            super().__init__()
            self.scale = nn.Parameter(torch.ones(E, 3, 1, 1))
            self.shift = nn.Parameter(torch.zeros(E, 3, 1, 1))
            self.gating = nn.Linear(16, E)

        def forward(self, priors, feats):
            return [p * self.scale + self.shift for p in priors], torch.log_softmax(self.gating(feats), 1)

    torch.manual_seed(0)
    nets = Nets().cuda()
    feats = torch.randn(B, 16, generator=torch.Generator().manual_seed(1)).cuda()
    priors = [c + 0.01 * torch.randn(c.shape, generator=torch.Generator().manual_seed(2 + b)).cuda() for b, c in enumerate(coords)]
    after, grads = [], []
    for batched in (True, False):
        m = copy.deepcopy(nets)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        opt.zero_grad()
        preds, lp = m(priors, feats)
        for p in preds:
            p.retain_grad()
        api.set_seed(77)
        if batched:
            losses = esac_loss_batch(preds, lp, assign, gts, *params)
            assert losses.shape == (B,)
            losses.sum().backward()
        else:
            sum(esac_loss(preds[b], lp[b], assign[b], gts[b], *per_image[b]) for b in range(B)).backward()
        grads.append([p.grad.clone() for p in preds])
        opt.step()
        after.append([p.detach().cpu().numpy() for p in m.parameters()])
    for ga, gb in zip(*grads):
        assert torch.equal(ga, gb)
    for a, b, p0 in zip(after[0], after[1], nets.parameters()):
        assert np.array_equal(a, b)
        assert not np.array_equal(a, p0.detach().cpu().numpy())


def test_loss_autograd_on_lists_gives_the_batch_mean_and_per_element_gradients(api):
    import torch
    from esac_b200.autograd import coord_loss, reproj_loss
    _, preds, gts = _reproj_inputs(900)
    ps = [torch.from_numpy(p).cuda().requires_grad_(True) for p in preds]
    loss = reproj_loss(ps, torch.from_numpy(gts).cuda(), 525.0, 0, 0, 10.0)
    (loss * 3.0).backward()
    B = len(preds)
    og = [torch.empty_like(p) for p in ps]
    per = api.reproj_loss([p.detach() for p in ps], torch.from_numpy(gts).cuda(), 525.0, 0, 0, 10.0, outGradients=og)
    assert loss.item() == torch.tensor(sum(per) / B, dtype=torch.float32).item()
    for p, g in zip(ps, og):
        assert torch.equal(p.grad, g * (torch.tensor(3.0, device="cuda") / B))
    qs = [torch.from_numpy(p).cuda().requires_grad_(True) for p in preds]
    tg = [(p.detach() + 0.3 * torch.randn_like(p)) for p in qs]
    loss = coord_loss(qs, tg, 1.0)
    loss.backward()
    per = api.coord_loss([q.detach() for q in qs], tg, 1.0, outGradients=og)
    assert loss.item() == torch.tensor(sum(per) / B, dtype=torch.float32).item()
    for q, g in zip(qs, og):
        assert torch.equal(q.grad, g * (torch.tensor(1.0, device="cuda") / B))


def test_ragged_example_runs_with_check():
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parents[1]
    r = subprocess.run([sys.executable, str(root / "examples" / "train_step_ragged_synthetic.py"), "--steps", "2", "--check"],
                       capture_output=True, text=True, cwd=root, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "check ok" in r.stdout
