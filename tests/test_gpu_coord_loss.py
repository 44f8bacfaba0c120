"""GPU tests of the fused scene-coordinate loss of the expert initialisation stage (init_expert.py:106-132; run with
`-m gpu`).

Tolerance: the yardstick is the float64 evaluation of the original op sequence (oracle/coord_loss_oracle.py), and the bar
is "at least as accurate as torch's own float32 evaluation": RMS deviation of the gradient from float64 within 1.5x of
torch-float32's, worst cell within 4x of torch-float32's worst cell, loss within 1e-6 relative.  The loss has a kink at
n = cutloss, where the gradient halves; a cell whose distance lies within rounding of the cut may land on either side in
any float32 evaluation, so cells within 1e-4 relative of the cut (by the float64 evaluation) are left out of the gradient
comparison and counted.  Cells with n == cut exactly and with d = 0 are checked on their own."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
CUT = 100.0


def _case(B, Hp, Wp, seed, Hg=None, Wg=None, invalid=0.0, offset=0.0, scale=2.0):
    """Ground truth around `offset` (world scale: ~500 m), a share `invalid` of all-zero ground-truth cells, and a
    prediction at log-uniform distances 1e-3..1e4 from it, so both branches of the loss get many cells.  Image 0 has a cell
    with d = 0 at (0, 0) and one with n == cut exactly at (0, 1)."""
    Hg, Wg = Hg or Hp, Wg or Wp
    rng = np.random.default_rng(seed)
    gt = (offset + scale * rng.standard_normal((B, 3, Hg, Wg))).astype(np.float32)
    gt = np.where(rng.random((B, 1, Hg, Wg)) < invalid, np.float32(0), gt)
    h, w = min(Hp, Hg), min(Wp, Wg)
    base = np.zeros((B, 3, Hp, Wp), np.float64)
    base[:, :, :h, :w] = gt[:, :, :h, :w]
    dist = 10.0 ** rng.uniform(-3, 4, (B, 1, Hp, Wp))
    dirn = rng.standard_normal((B, 3, Hp, Wp))
    pred = (base + dist * dirn / np.linalg.norm(dirn, axis=1, keepdims=True)).astype(np.float32)
    c = np.float32(offset) + np.array([1.0, 2.0, 3.0], np.float32)
    gt[0, :, 0, 0] = pred[0, :, 0, 0] = c                 # d = 0
    gt[0, :, 0, 1] = c
    pred[0, :, 0, 1] = c + np.array([0.0, 0.0, CUT], np.float32)   # n == cut (exact in float32)
    assert pred[0, 2, 0, 1] - gt[0, 2, 0, 1] == CUT
    return pred, gt


def _run(pred, gt, dev="cuda", grads=True, cut=CUT):
    import torch
    import esac_b200.api as api
    p = torch.from_numpy(pred).to(dev)
    q = torch.from_numpy(gt).to(dev)
    g = torch.full(p.shape, 7.0, device=dev) if grads else None      # prefilled: must be overwritten
    losses, counts = api.coord_loss(p, q, cut, outGradients=g, return_counts=True)
    return np.array(losses), counts, (g.cpu().numpy() if grads else None)


def _check_against_oracle(pred, gt, losses, counts, g, cut=CUT):
    import torch
    from oracle.coord_loss_oracle import coord_loss_and_grad
    B, _, Hp, Wp = pred.shape
    Hg, Wg = gt.shape[2:]
    h, w = min(Hp, Hg), min(Wp, Wg)
    for b in range(B):
        l32, g32 = coord_loss_and_grad(torch.from_numpy(pred[b]), torch.from_numpy(gt[b]), cut)
        l64, g64 = coord_loss_and_grad(torch.from_numpy(pred[b]), torch.from_numpy(gt[b]), cut, dtype=torch.float64)
        assert abs(losses[b] - l64) <= 1e-6 * max(1.0, abs(l64)), (b, losses[b], l32, l64)
        valid = np.abs(gt[b, :, :h, :w]).sum(0) != 0
        assert counts[b] == int(valid.sum())
        n64 = np.linalg.norm(pred[b, :, :h, :w].astype(np.float64) - gt[b, :, :h, :w].astype(np.float64), axis=0)
        kink = np.zeros((Hp, Wp), bool)
        kink[:h, :w] = valid & (np.abs(n64 - cut) <= 1e-4 * cut)
        assert kink.sum() <= 2e-4 * h * w + 2, kink.sum()
        keep = ~kink[None]
        g64 = g64.numpy()
        d32 = (g32.double().numpy() - g64) * keep
        dk = (g[b] - g64) * keep
        scale = np.abs(g64).max()
        rms_k, rms_32 = np.sqrt((dk ** 2).mean()), np.sqrt((d32 ** 2).mean())
        assert rms_k <= 1.5 * rms_32 + 1e-7 * scale, (b, rms_k, rms_32, scale)
        assert np.abs(dk).max() <= 4 * np.abs(d32).max() + 1e-6 * scale, (b, np.abs(dk).max(), np.abs(d32).max(), scale)
        # outside the window and on invalid cells the gradient is exactly zero
        outside = np.ones((Hp, Wp), bool)
        outside[:h, :w] = ~valid
        assert (g[b][:, outside] == 0).all()


CASES = {
    "1x60x80_half_invalid": dict(B=1, Hp=60, Wp=80, invalid=0.5),
    "3x60x80_half_invalid": dict(B=3, Hp=60, Wp=80, invalid=0.5),
    "2x33x47_scalar_path": dict(B=2, Hp=33, Wp=47),
    "2x80x60": dict(B=2, Hp=80, Wp=60),
    "1x480x640": dict(B=1, Hp=480, Wp=640),
    "2x60x80_world_scale": dict(B=2, Hp=60, Wp=80, offset=500.0, scale=30.0, invalid=0.2),
}


@pytest.mark.parametrize("name", list(CASES))
def test_coord_loss_matches_float64_oracle(name):
    kw = dict(CASES[name])
    pred, gt = _case(seed=100 + list(CASES).index(name), **kw)
    losses, counts, g = _run(pred, gt)
    _check_against_oracle(pred, gt, losses, counts, g)
    # d = 0: zero gradient; n == cut: the L1 branch, gradient d / n / count = 1 / count on z
    assert (g[0, :, 0, 0] == 0).all()
    assert g[0, 0, 0, 1] == 0 and g[0, 1, 0, 1] == 0
    assert g[0, 2, 0, 1] == np.float32(1.0 / counts[0])


def test_mask_counts_any_nonzero_component():
    """gt.abs().sum(0) != 0: a cell with only x, only y or only z nonzero is valid, a subnormal component too, and so is
    a NaN one (it counts, adds nothing to the loss, and its gradient is NaN)."""
    pred, gt = _case(2, 60, 80, seed=61)
    keep = np.random.default_rng(62).random(gt.shape) < 0.4      # components zeroed independently
    gt = np.where(keep, gt, np.float32(0))
    gt[1, :, 5, :10] = 0.0
    gt[1, 0, 5, :5] = np.float32(1e-40)                          # subnormal x only
    gt[1, 1, 5, 5:10] = np.float32(-1e-42)                       # subnormal y only
    gt[0, :, 3, 3] = 0.0
    single = (gt != 0).sum(1) == 1
    assert single.sum() > 1000 and (single & (gt[:, 2] == 0)).sum() > 1000
    losses, counts, g = _run(pred, gt)
    _check_against_oracle(pred, gt, losses, counts, g)
    assert counts == [int(v) for v in (np.abs(gt).sum(1) != 0).sum((1, 2))]
    assert (g[1, :, 5, :10] != 0).all()
    gt[0, :, 3, 3] = [np.nan, 0.0, 0.0]                          # a NaN ground-truth cell where there was none
    l_nan, c_nan, g_nan = _run(pred, gt)
    assert c_nan == [counts[0] + 1, counts[1]]
    assert np.isnan(g_nan[0, :, 3, 3]).all()
    assert l_nan[0] == pytest.approx(losses[0] * counts[0] / (counts[0] + 1), rel=1e-12) and l_nan[1] == losses[1]


def test_known_answer_on_device():
    """cut = 100, four valid cells: d = 0, NaN prediction, n = 100, n = 400; one invalid cell."""
    gt = np.zeros((1, 3, 1, 5), np.float32)
    pred = np.zeros((1, 3, 1, 5), np.float32)
    gt[0, :, 0, 0] = pred[0, :, 0, 0] = [1.0, 2.0, 3.0]
    gt[0, :, 0, 1] = [1.0, 2.0, 3.0]
    pred[0, :, 0, 1] = np.nan
    gt[0, 2, 0, 2], pred[0, 2, 0, 2] = 5.0, 105.0
    gt[0, 2, 0, 3], pred[0, 2, 0, 3] = 5.0, 405.0
    pred[0, :, 0, 4] = 7.0
    for dev in ("cpu", "cuda"):
        losses, counts, g = _run(pred, gt, dev)
        assert losses[0] == 75.0 and counts == [4]
        np.testing.assert_array_equal(g[0, 2, 0], np.array([0.0, np.nan, 0.25, 0.0625, 0.0], np.float32))
        assert np.isnan(g[0, :, 0, 1]).all()
        assert (g[0, :2, 0, [0, 2, 3, 4]] == 0).all()


@pytest.mark.parametrize("pred_hw,gt_hw", [((61, 81), (60, 80)), ((60, 80), (61, 81)), ((61, 80), (60, 81)),
                                           ((60, 81), (61, 80)),
                                           ((61, 80), (60, 80)), ((60, 80), (61, 80))])   # equal widths: 128-bit path
def test_crop_to_the_common_window(pred_hw, gt_hw):
    pred, gt = _case(2, *pred_hw, seed=77, Hg=gt_hw[0], Wg=gt_hw[1], invalid=0.3)
    losses, counts, g = _run(pred, gt)
    _check_against_oracle(pred, gt, losses, counts, g)
    h, w = min(pred_hw[0], gt_hw[0]), min(pred_hw[1], gt_hw[1])
    assert (g[:, :, h:, :] == 0).all() and (g[:, :, :, w:] == 0).all()


def test_size_difference_of_two_is_an_error():
    import esac_b200.api as api
    pred, gt = _case(1, 62, 80, seed=3, Hg=60, Wg=80)
    with pytest.raises(RuntimeError, match="size mismatch"):
        api.coord_loss(pred, gt)
    with pytest.raises(RuntimeError, match="size mismatch"):
        api.coord_loss(np.ascontiguousarray(pred[:, :, :60]), np.zeros((1, 3, 60, 82), np.float32))
    # the C ABI checks it too, with a negative status and a message
    ctx = api.context()
    losses = np.zeros(1)
    rc = ctx.lib.esacb200_coord_loss(ctx.handle, 1, pred.ctypes.data, 62, 80, gt.ctypes.data, 60, 80, None, 100.0,
                                     losses.ctypes.data, None)
    assert rc == -2 and b"size mismatch" in ctx.lib.esacb200_last_error(ctx.handle)
    rc = ctx.lib.esacb200_coord_loss(ctx.handle, 1, None, 60, 80, gt.ctypes.data, 60, 80, None, 100.0, losses.ctypes.data, None)
    assert rc == -2 and b"null" in ctx.lib.esacb200_last_error(ctx.handle)
    rc = ctx.lib.esacb200_coord_loss(ctx.handle, 0, pred.ctypes.data, 60, 80, gt.ctypes.data, 60, 80, None, 100.0,
                                     losses.ctypes.data, None)
    assert rc == -2 and b"bad sizes" in ctx.lib.esacb200_last_error(ctx.handle)


@pytest.mark.parametrize("shape", [(2, 60, 80), (1, 480, 640), (2, 60, 81)])
def test_aligned_and_misaligned_views_agree_bitwise(shape):
    import torch
    import esac_b200.api as api
    B, H, W = shape
    pred, gt = _case(B, H, W, seed=11, invalid=0.4)
    n = pred.size
    results = []
    for shift in (0, 1):   # shift 1: every map starts 4 bytes past a 16-byte boundary -> scalar loads
        bufs = [torch.zeros(n + 4, device="cuda") for _ in range(3)]
        p = bufs[0][shift:shift + n].view(pred.shape)
        q = bufs[1][shift:shift + n].view(gt.shape)
        g = bufs[2][shift:shift + n].view(pred.shape)
        p.copy_(torch.from_numpy(pred))
        q.copy_(torch.from_numpy(gt))
        assert (p.data_ptr() % 16 == 0) == (shift == 0)
        losses = api.coord_loss(p, q, CUT, outGradients=g)
        results.append((losses, g.cpu().numpy()))
    assert results[0][0] == results[1][0]
    np.testing.assert_array_equal(results[0][1], results[1][1])


def test_call_behaviour():
    import torch
    import esac_b200.api as api
    pred, gt = _case(3, 60, 80, seed=21, invalid=0.5)
    gt[1] = 0.0                                                     # image 1: no valid cell
    l_cuda, c_cuda, g_cuda = _run(pred, gt, "cuda")
    l_cpu, c_cpu, g_cpu = _run(pred, gt, "cpu")
    l_again, _, g_again = _run(pred, gt, "cuda")
    # host and device inputs, and two calls, agree bit for bit
    assert l_cuda.tobytes() == l_cpu.tobytes() == l_again.tobytes() and c_cuda == c_cpu
    assert g_cuda.tobytes() == g_cpu.tobytes() == g_again.tobytes()
    # the prefilled 7.0 is gone everywhere
    assert not (g_cuda == 7.0).any()
    # loss only: the same losses
    l_only, c_only, _ = _run(pred, gt, "cuda", grads=False)
    assert l_only.tobytes() == l_cuda.tobytes() and c_only == c_cuda
    assert np.array(api.coord_loss(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), CUT)).tobytes() == l_cuda.tobytes()
    # no valid cell: NaN loss, zero gradient; the other images are what they are on their own
    assert np.isnan(l_cuda[1]) and c_cuda[1] == 0 and (g_cuda[1] == 0).all()
    for b in (0, 2):
        lb, cb, gb = _run(pred[b:b + 1], gt[b:b + 1], "cuda")
        assert lb[0] == l_cuda[b] and cb[0] == c_cuda[b] and gb[0].tobytes() == g_cuda[b].tobytes()
    _check_against_oracle(pred[[0, 2]], gt[[0, 2]], l_cuda[[0, 2]], [c_cuda[0], c_cuda[2]], g_cuda[[0, 2]])


def test_non_default_stream_orders_after_the_producer():
    import torch
    import esac_b200.api as api
    pred, gt = _case(2, 120, 160, seed=31, invalid=0.3)
    ref_l, _, ref_g = _run(pred, gt, "cuda")
    src_p, src_q = torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()
    big = torch.randn(4096, 4096, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        p = torch.zeros_like(src_p)
        q = torch.zeros_like(src_q)
        g = torch.full_like(src_p, 7.0)
        for _ in range(40):                          # ~10 ms of queued work ahead of the real inputs
            big = big @ big * 1e-3
        p.copy_(src_p)
        q.copy_(src_q)
        losses = api.coord_loss(p, q, CUT, outGradients=g)
        g_host = g.cpu().numpy()
    assert np.array(losses).tobytes() == ref_l.tobytes()
    assert g_host.tobytes() == ref_g.tobytes()


def test_one_adam_step_matches_the_float64_op_sequence():
    import torch
    pred, gt = _case(1, 61, 81, seed=41, Hg=60, Wg=80, invalid=0.5)
    prior = torch.from_numpy(pred)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the stand-in expert runs in true float32
    try:
        _adam_step(prior, gt)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _adam_step(prior, gt):
    import torch
    import torch.nn as nn
    from esac_b200.autograd import coord_loss
    from oracle.coord_loss_oracle import coord_loss as original
    models, opts = [], []
    for dtype, dev in ((torch.float32, "cuda"), (torch.float64, "cpu")):
        torch.manual_seed(0)
        m = nn.Conv2d(3, 3, 1).to(dtype=dtype, device=dev)
        with torch.no_grad():
            m.weight.copy_(torch.eye(3).view(3, 3, 1, 1) + 0.01 * torch.randn(3, 3, 1, 1))
            m.bias.fill_(0.1)
        models.append(m)
        opts.append(torch.optim.Adam(m.parameters(), lr=1e-4))
    loss = coord_loss(models[0](prior.cuda()), torch.from_numpy(gt).cuda(), CUT)
    (loss * 2.0).backward()
    ref = original(models[1](prior.double()), torch.from_numpy(gt), CUT, dtype=torch.float64)
    (ref * 2.0).backward()
    assert abs(loss.item() - ref.item()) <= 1e-6 * max(1.0, abs(ref.item()))
    for a, r in zip(models[0].parameters(), models[1].parameters()):
        assert (a.grad.cpu().double() - r.grad).abs().max().item() <= 1e-5 * r.grad.abs().max().item()
    for o in opts:
        o.step()
    for a, r in zip(models[0].parameters(), models[1].parameters()):
        # the step moves every parameter by ~lr = 1e-4; what is left is float32 rounding of parameters of size ~1
        assert (a.detach().cpu().double() - r.detach()).abs().max().item() <= 2.5e-7


def test_mean_over_a_batch_is_the_autograd_loss():
    import torch
    from esac_b200.autograd import coord_loss
    pred, gt = _case(3, 60, 80, seed=51, invalid=0.5)
    losses, _, g = _run(pred, gt)
    p = torch.from_numpy(pred).cuda().requires_grad_(True)
    loss = coord_loss(p, torch.from_numpy(gt).cuda(), CUT)
    loss.backward()
    assert loss.item() == pytest.approx(float(np.mean(losses)), rel=1e-6)
    np.testing.assert_array_equal(p.grad.cpu().numpy(), g * (np.float32(1.0) / np.float32(3)))   # grads * (grad_out / B)


def test_init_expert_example_runs_with_check():
    r = subprocess.run([sys.executable, str(ROOT / "examples" / "init_expert_step_synthetic.py"), "--iterations", "3", "--check"],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("Iteration:") == 3
