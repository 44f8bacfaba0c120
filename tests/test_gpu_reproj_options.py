"""The fused reprojection loss (api.reproj_loss / reproj_loss_async, reproj.cu) at every option, launch shape and kink
(run with `-m gpu`).

The bar is tests/test_gpu_reproj.py's, against the float64 evaluation of the same op sequence: the loss within 1e-5,
the RMS gradient error within 1.5x of torch float32's, the worst cell within 4x of torch float32's worst -- or, cell by
cell, within 4x of what float32 can promise for that cell.  That promise is 16 ulp of the cell's gradient plus the
conditioning of its error direction: the float32 rounding of its pixel error (~16 ulp of the largest terms of the
transform and projection -- f times the world and camera coordinates, cx*zc -- divided by the depth; it grows behind
the camera and near minDepth, where those terms cancel and are divided by minDepth) over the error itself.  The second
form matters where torch float32 is correctly rounded to an ulp and the kernel's rcp.approx / rsqrt.approx add a few,
and where a handful of ill-conditioned cells would decide a comparison with torch by luck.  Cells within 1e-3 px plus
that rounding of the call's own cut or maxReproj, or with a depth within 2e-5 of its minDepth, may land on either side
of the kink in any float32 evaluation and are left out of the gradient comparison (and counted).

  * options: maxReproj in {100, 30, 250, 5 < cut}, minDepth in {0.1, 0.01, 1, 2.5}, subSampling in {1, 3, 4, 8}, on
    scenes whose errors and depths straddle each of them, on both load paths, eager and stream-ordered (bitwise equal);
  * single-cell probes (tests/test_reproj_oracle_options.py): cut +- 1e-4 px, maxReproj +- 1e-3 px, depth at minDepth and
    one float32 ulp either side, behind the camera, on target, NaN, float32 overflow -- each against float64 at 1e-5;
  * launch shapes at both boundaries of each range of reproj_blocks_per_image (63, 64, 65, 255 and 256 blocks of cells),
    each with an odd-sized scalar-path twin, ragged, stacked B = 64, through coord_loss too (same rule, same reduction),
    and a captured ragged call that needs reproj_max_blocks' workspace."""
import math

import numpy as np
import pytest
import torch

import esac_b200.api as api
from oracle.reproj_loss_oracle import reproj_errors, reproj_loss_and_grad
from test_reproj_oracle_options import (F_PROBE, PROBES, PROBE_OPTIONS, camera_coords, f32, probe_image, probe_reference,
                                        straddling_scene)

pytestmark = pytest.mark.gpu

CUT = 10.0


def _check_image(pred, gt, f, padx, pady, ppx, ppy, sub, cut, max_reproj, min_depth, loss, grad):
    """One image of a kernel call against float64 (and torch float32 as the bar)."""
    kw = dict(image_w=2 * ppx, image_h=2 * ppy, max_reproj=max_reproj, min_depth=min_depth)
    t_pred, t_gt = torch.from_numpy(pred), torch.from_numpy(gt)
    l32, g32 = reproj_loss_and_grad(t_pred, t_gt, f, padx, pady, cut, sub, **kw)
    l64, g64 = reproj_loss_and_grad(t_pred, t_gt, f, padx, pady, cut, sub, dtype=torch.float64, **kw)
    assert abs(loss - l64) <= 1e-5 * max(1.0, abs(l64)), (loss, l32, l64)
    e64 = reproj_errors(t_pred, t_gt, f, padx, pady, sub, dtype=torch.float64, **dict(kw, max_reproj=math.inf)).numpy()
    xc, yc, zc = camera_coords(pred, gt)
    world = np.abs(pred.reshape(3, -1).astype(np.float64)).max(0) + np.abs(gt[:3, 3]).max()
    rounding = 1e-6 * (f * (world + np.maximum(np.abs(xc), np.abs(yc))) + max(ppx, ppy) * np.abs(zc)) / np.maximum(zc, min_depth)
    margin = 1e-3 + rounding
    kink = (np.abs(e64 - cut) < margin) | (np.abs(e64 - max_reproj) < margin) | (np.abs(zc - min_depth) < 2e-5)
    n = e64.size
    assert kink.sum() <= 2e-3 * n + 4, kink.sum()
    keep = ~kink.reshape(1, *pred.shape[1:])
    g64 = g64.numpy()
    scale = np.abs(g64).max()
    d32 = np.abs(g32.double().numpy() - g64).reshape(3, -1).max(0)[keep.reshape(-1)]
    dk = np.abs(grad - g64).reshape(3, -1).max(0)[keep.reshape(-1)]
    promise = (np.abs(g64).reshape(3, -1).max(0) * (rounding / np.maximum(e64, 1e-30) + 1e-6))[keep.reshape(-1)]
    worst = np.maximum(4 * d32.max(), 4 * promise) + 1e-6 * scale
    assert (dk <= worst).all(), (dk.max(), d32.max(), np.argmax(dk / worst), scale)
    rms_k, rms_32, rms_p = (np.sqrt((v ** 2).sum() / n) for v in (dk, d32, promise))
    assert rms_k <= 1.5 * rms_32 + rms_p + 1e-7 * scale, (rms_k, rms_32, rms_p, scale)


def _run(scenes, sub, cut, max_reproj, min_depth, fill=7.0):
    """Eager and stream-ordered ragged calls on the scenes: (losses, gradients as numpy), the second bitwise the first."""
    preds = [torch.from_numpy(s[0]).cuda() for s in scenes]
    gts = torch.from_numpy(np.stack([s[1] for s in scenes])).cuda()
    f, px, py, cx, cy = ([s[i] for s in scenes] for i in range(2, 7))
    grads = [torch.full_like(p, fill) for p in preds]
    losses = api.reproj_loss(preds, gts, f, px, py, cut, sub, cx, cy, outGradients=grads, maxReproj=max_reproj,
                             minDepth=min_depth)
    B = len(scenes)
    shifts = torch.tensor([[a, b] for a, b in zip(px, py)], dtype=torch.int32, device="cuda")
    cams = torch.tensor([[a, b, c] for a, b, c in zip(f, cx, cy)], dtype=torch.float32, device="cuda")
    a_losses = torch.full((B,), -1.0, dtype=torch.float64, device="cuda")
    a_status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    a_grads = [torch.full_like(p, -fill) for p in preds]
    api.reproj_loss_async(preds, gts, shifts, cams, cut, sub, a_losses, a_status, outGradients=a_grads, maxReproj=max_reproj,
                          minDepth=min_depth)
    torch.cuda.synchronize()
    assert a_status.tolist() == [0] * B
    assert np.array(losses).tobytes() == a_losses.cpu().numpy().tobytes()
    g = [x.cpu().numpy() for x in grads]
    for x, y in zip(g, a_grads):
        assert x.tobytes() == y.cpu().numpy().tobytes()
    return losses, g


# ---- options grid -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sub", [1, 3, 4, 8])
@pytest.mark.parametrize("min_depth", [0.1, 0.01, 1.0, 2.5])
@pytest.mark.parametrize("max_reproj", [100.0, 30.0, 250.0, 5.0])
def test_options_match_float64(max_reproj, min_depth, sub):
    """A 24x32 map (vector path) and a 23x31 one (scalar path) in one ragged call."""
    seed = int(max_reproj * 7 + min_depth * 100 + sub)
    scenes = [straddling_scene(24, 32, sub, seed, CUT, max_reproj, min_depth),
              straddling_scene(23, 31, sub, seed + 1, CUT, max_reproj, min_depth)]
    losses, grads = _run(scenes, sub, CUT, max_reproj, min_depth)
    for s, loss, g in zip(scenes, losses, grads):
        _check_image(*s, sub, CUT, max_reproj, min_depth, loss, g)


# ---- single-cell probes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cut,max_reproj,min_depth", PROBE_OPTIONS)
def test_single_cell_probes(cut, max_reproj, min_depth):
    """One probe per image, on an 8x12 map (vector path, the probe in each lane of a 4-cell group in turn) and a 7x11 one
    (scalar path); every other cell's gradient is exactly 0, the probe's is float64's within 1e-5."""
    cut, max_reproj, min_depth = f32(cut, max_reproj, min_depth)
    sub = 8
    images = []
    for k, probe in enumerate(PROBES):
        for H, W in ((8, 12), (7, 11)):
            cell = (13 + 7 * k) % (H * W)
            pred, ppx, ppy = probe_image(H, W, sub, cell, probe, cut, max_reproj, min_depth)
            images.append((probe, cell, (pred, np.eye(4, dtype=np.float32), F_PROBE, 0, 0, ppx, ppy)))
    losses, grads = _run([im[2] for im in images], sub, cut, max_reproj, min_depth)
    for (probe, cell, s), loss, g in zip(images, losses, grads):
        l64, g64, _ = probe_reference(s[0], sub, s[5], s[6], cut, max_reproj, min_depth)
        assert abs(loss - l64) <= 1e-5 * max(1.0, abs(l64)), (probe, loss, l64)
        g, g64 = g.reshape(3, -1), g64.reshape(3, -1)
        others = np.arange(g.shape[1]) != cell
        assert (g[:, others] == 0).all(), probe
        gc, rc = g[:, cell], g64[:, cell]
        if probe == "nan":
            assert np.isnan(gc).all() and np.isnan(rc).all()
        elif (rc == 0).all():             # beyond maxReproj, on target, or overflowing float32 (not float64)
            assert (gc == 0).all(), (probe, gc)
        else:
            assert np.abs(gc - rc).max() <= 1e-5 * np.abs(rc).max(), (probe, gc, rc)


# ---- launch shapes ------------------------------------------------------------------------------------------------------
# 1024-cell blocks: 63 (one pass per CTA), 64 and 65 (two passes), 255 (two), 256 (four); vector-path maps and odd twins
SHAPES = {63: [(63, 1024), (251, 257)], 64: [(256, 256), (255, 257)], 65: [(145, 452), (257, 257)],
          255: [(510, 512), (509, 511)], 256: [(512, 512), (511, 513)]}
ALL_SHAPES = [s for v in SHAPES.values() for s in v]


def _scene(shape, seed, sub=1):
    return straddling_scene(*shape, sub, seed, CUT, 100.0, 0.1)


@pytest.mark.parametrize("need", list(SHAPES))
def test_block_rule_boundaries_match_float64(need):
    for i, shape in enumerate(SHAPES[need]):
        H, W = shape
        assert (H * W + 1023) // 1024 == need and (H * W % 4 == 0) == (i == 0)
        s = _scene(shape, need * 10 + i)
        losses, grads = _run([s], 1, CUT, 100.0, 0.1, fill=float("nan"))
        _check_image(*s, 1, CUT, 100.0, 0.1, losses[0], grads[0])


def test_ragged_mix_of_all_shapes_is_each_image_alone():
    """grid.x is the largest image's block count; the smaller images leave their extra blocks at once."""
    scenes = [_scene(shape, 500 + i) for i, shape in enumerate(ALL_SHAPES)]
    losses, grads = _run(scenes, 1, CUT, 100.0, 0.1)
    for s, loss, g in zip(scenes, losses, grads):
        l1, g1 = _run([s], 1, CUT, 100.0, 0.1)
        assert l1[0] == loss and g1[0].tobytes() == g.tobytes()


def test_stacked_batch_of_64():
    B, H, W, sub = 64, 60, 80, 8
    scenes = [straddling_scene(H, W, sub, 900 + b, CUT, 100.0, 0.1) for b in range(B)]
    preds = torch.from_numpy(np.stack([s[0] for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s[1] for s in scenes])).cuda()
    f, px, py, cx, cy = ([s[i] for s in scenes] for i in range(2, 7))
    grads = torch.full_like(preds, float("nan"))
    losses = api.reproj_loss(preds, gts, f, px, py, CUT, sub, cx, cy, outGradients=grads)
    g = grads.cpu().numpy()
    for b, s in enumerate(scenes):
        _check_image(*s, sub, CUT, 100.0, 0.1, losses[b], g[b])


@pytest.mark.parametrize("need", list(SHAPES))
def test_coord_loss_block_rule_boundaries_match_float64(need):
    from test_gpu_coord_loss import _case, _check_against_oracle, _run as coord_run
    preds, gts, singles = [], [], []
    for i, (H, W) in enumerate(SHAPES[need]):
        pred, gt = _case(1, H, W, 40 + need + i, invalid=0.2)
        losses, counts, g = coord_run(pred, gt)
        _check_against_oracle(pred, gt, losses, counts, g)
        preds.append(pred[0]); gts.append(gt[0]); singles.append((losses[0], g[0]))
    # both shapes in one ragged call: each bitwise its own call
    p = [torch.from_numpy(x).cuda() for x in preds]
    q = [torch.from_numpy(x).cuda() for x in gts]
    og = [torch.full_like(x, 7.0) for x in p]
    losses = api.coord_loss(p, q, 100.0, outGradients=og)
    for (l1, g1), loss, g in zip(singles, losses, og):
        assert l1 == loss and g1.tobytes() == g.cpu().numpy().tobytes()


def test_captured_ragged_call_fits_the_reserved_workspace():
    """reserve_loss_async(2, 256, 256) then a captured ragged call of two maps of 63x1024 cells each (one per load path):
    63 blocks each, more than the 32 of a 256x256 map, which reproj_max_blocks reserves for.  The replay is bitwise the
    eager call."""
    saved = api._contexts.get(0)
    ctx = api.Context(0)                  # a workspace that has seen only this test
    api._contexts[0] = ctx
    try:
        scenes = [_scene((63, 1024), 71), _scene((251, 257), 72)]
        api.reserve_loss_async(2, 256, 256)
        preds = [torch.from_numpy(s[0]).cuda() for s in scenes]
        gts = torch.from_numpy(np.stack([s[1] for s in scenes])).cuda()
        shifts = torch.tensor([[s[3], s[4]] for s in scenes], dtype=torch.int32, device="cuda")
        cams = torch.tensor([[s[2], s[5], s[6]] for s in scenes], dtype=torch.float32, device="cuda")
        grads = [torch.full_like(p, 7.0) for p in preds]
        losses = torch.zeros(2, dtype=torch.float64, device="cuda")
        status = torch.full((2,), -1, dtype=torch.int32, device="cuda")
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            api.reproj_loss_async(preds, gts, shifts, cams, CUT, 1, losses, status, outGradients=grads)
        graph.replay()
        torch.cuda.synchronize()
        ref_g = [torch.zeros_like(p) for p in preds]
        ref = api.reproj_loss(preds, gts, [s[2] for s in scenes], [s[3] for s in scenes], [s[4] for s in scenes], CUT, 1,
                              [s[5] for s in scenes], [s[6] for s in scenes], outGradients=ref_g)
        assert status.tolist() == [0, 0]
        assert losses.cpu().numpy().tobytes() == np.array(ref).tobytes()
        for g, r in zip(grads, ref_g):
            assert g.cpu().numpy().tobytes() == r.cpu().numpy().tobytes()
    finally:
        torch.cuda.synchronize()
        if saved is not None:
            api._contexts[0] = saved
        else:
            api._contexts.pop(0, None)
        ctx.close()
