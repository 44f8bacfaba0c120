"""Each batched entry point makes one call, to the library's ragged form, whether its images come as one stacked tensor or
as a list; a stacked tensor and the list of its slices hand the library the same pointers, sizes, shifts and cameras.
The library is a stub here (no context, no device): it records every call and, for the autograd nodes, writes known
losses and gradients through the host pointers it is given."""
import ctypes as C

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import autograd
from esac_b200.synth import make_scene

B, E, H, W, M = 3, 2, 8, 10, 4
TAIL = (10.0, 100.0, 0.5, 100.0, 8)
CAMS = ([3, -1, 0], [2, 0, -4], [525.3, 1e-3 + 1 / 3, 2 ** 24 + 1.0], [40.0, 41.5, 39.25], [32.0, 30.5, 33.75])
# argument index of shiftX in each entry point that takes shifts and cameras; shiftY, f, ppx, ppy follow
CAM_AT = {"esacb200_forward_ragged": 10, "esacb200_backward_ragged": 14, "esacb200_reproj_loss_ragged": 7,
          "esacb200_hypotheses_forward_ragged": 9}


class Call:
    def __init__(self, name, args):
        self.name, self.args = name, args
        # what the pointer and size arrays hold during the call (the camera arrays die with it)
        self.arrays = {i: list(a) for i, a in enumerate(args) if isinstance(a, C.Array)}
        at = CAM_AT.get(name)
        self.cams = None if at is None else [C.string_at(args[at + k], 4 * args[1]) for k in range(5)]


class Lib:
    def __init__(self):
        self.calls, self.fill = [], {}

    def __getattr__(self, name):
        def entry(*args):
            self.calls.append(Call(name, args))
            if name in self.fill:
                self.fill[name](args)
            return 0
        return entry


class Ctx:
    handle, device = None, 0

    def __init__(self):
        self.lib = Lib()

    def check(self, rc):
        assert rc == 0

    def set_stream(self, stream):
        pass


@pytest.fixture
def ctx(monkeypatch):
    stub = Ctx()
    monkeypatch.setattr(api, "_pick_ctx", lambda *devices: stub)
    # the hypotheses node allocates its tapes on torch's CUDA device; without one they are host tensors
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, device=None, **k: empty(*a, **k))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: type("Stream", (), {"cuda_stream": 0}))
    monkeypatch.setattr(api, "_tape_hypotheses", lambda t, E, H, W, what: M)
    return stub


@pytest.fixture(scope="module")
def batch():
    scenes = [make_scene(E=E, H=H, W=W, M=M, seed=b) for b in range(B)]
    coords = torch.from_numpy(np.stack([s.coords for s in scenes]))
    pred = coords[:, 0].contiguous()
    return {"coords": coords, "assign": torch.from_numpy(np.stack([s.assign for s in scenes])),
            "gts": torch.from_numpy(np.stack([s.gt_pose for s in scenes])), "grads": torch.zeros_like(coords), "pred": pred,
            "gt_coords": pred + 1.0, "pred_grads": torch.zeros_like(pred), "poses": torch.zeros(B, 4, 4),
            "tapes": [torch.zeros(16, dtype=torch.uint8) for _ in range(B)]}


def _calls(t, form, cams=CAMS):
    """Every batched entry point once, on the stacked tensors or on the lists of their slices."""
    s = (lambda x: list(t[x].unbind(0))) if form == "list" else (lambda x: t[x])
    return {
        "esacb200_forward_ragged": lambda: api.forward_batch(s("coords"), t["assign"], t["poses"], *cams, *TAIL),
        "esacb200_backward_ragged": lambda: api.backward_batch(s("coords"), s("grads"), t["assign"], t["gts"], 1.0, 100.0,
                                                                100.0, *cams, *TAIL),
        "esacb200_reproj_loss_ragged": lambda: api.reproj_loss(s("pred"), t["gts"], cams[2], cams[0], cams[1], 10.0, 8, cams[3],
                                                               cams[4], outGradients=s("pred_grads")),
        "esacb200_coord_loss_ragged": lambda: api.coord_loss(s("pred"), s("gt_coords"), 10.0, outGradients=s("pred_grads")),
        "esacb200_hypotheses_forward_ragged": lambda: api.hypotheses_forward_batch(s("coords"), t["assign"], *cams, *TAIL),
        "esacb200_hypotheses_backward_ragged": lambda: api.hypotheses_backward_batch(t["tapes"], s("coords"), s("grads")),
    }


@pytest.mark.parametrize("form", ["stacked", "list"])
def test_each_batched_call_is_one_call_of_the_ragged_entry_point(ctx, batch, form):
    for name, call in _calls(batch, form).items():
        ctx.lib.calls.clear()
        call()
        assert [c.name for c in ctx.lib.calls] == [name]


def test_a_stacked_tensor_and_the_list_of_its_slices_hand_over_the_same_arrays(ctx, batch):
    seen = {}
    for form in ("stacked", "list"):
        for name, call in _calls(batch, form).items():
            ctx.lib.calls.clear()
            call()
            (c,) = ctx.lib.calls
            seen.setdefault(name, []).append(c)
    for c in seen["esacb200_hypotheses_forward_ragged"]:
        del c.arrays[19]   # the tapes, which each call allocates
    for name, (stacked, listed) in seen.items():
        # the pointer arrays of every image argument, the heights and widths
        assert stacked.arrays and stacked.arrays == listed.arrays, name
        assert stacked.cams == listed.cams, name
    # image b of a stacked tensor starts b images past its base
    fwd = seen["esacb200_forward_ragged"][0]
    base = batch["coords"].data_ptr()
    assert fwd.arrays[2] == [base + b * E * 3 * H * W * 4 for b in range(B)]
    assert fwd.arrays[3] == [H] * B and fwd.arrays[4] == [W] * B


def _floats(values, ctype):
    return bytes((ctype * B)(*values))


def test_scalar_cameras_are_broadcast_as_ctypes_rounds_them(ctx, batch):
    one = (3, -2, 525.3, 1e-3 + 1 / 3, 583.2999999999)
    for name, call in _calls(batch, "stacked", cams=one).items():
        if name not in CAM_AT:
            continue
        ctx.lib.calls.clear()
        call()
        (c,) = ctx.lib.calls
        want = [_floats([v] * B, C.c_int if k < 2 else C.c_float) for k, v in enumerate(one)]
        assert c.cams == want, name
    # the reprojection loss's default principal point: each image's own centre of its sub*W x sub*H frame
    sizes = [(8, 10), (7, 12), (9, 9)]
    pred = [torch.zeros(3, h, w) for h, w in sizes]
    ctx.lib.calls.clear()
    api.reproj_loss(pred, batch["gts"], 525.0, 0, 0, 10.0, 8)
    (c,) = ctx.lib.calls
    assert c.cams[3] == _floats([w * 4.0 for _, w in sizes], C.c_float)
    assert c.cams[4] == _floats([h * 4.0 for h, _ in sizes], C.c_float)


# ---- the autograd nodes on a stub that writes known losses and gradients ---------------------------------------------
def _pattern(b, n):
    return ((b + 1) + np.arange(n) / n).astype(np.float32)


def _write_images(ptrs, sizes):
    for b, (p, n) in enumerate(zip(ptrs, sizes)):
        values = _pattern(b, n)
        C.memmove(p, values.ctypes.data, 4 * n)


def _write_losses(ptr):
    values = np.arange(1.0, B + 1.0)
    C.memmove(ptr, values.ctypes.data, 8 * B)


def _expected(like, scale):
    """The gradients the stub writes, each times image b's factor, in the shape of `like`'s images."""
    return [torch.from_numpy(_pattern(b, t.numel())).reshape(t.shape) * scale[b] for b, t in enumerate(like)]


@pytest.fixture
def filled(ctx):
    ctx.lib.fill = {
        "esacb200_backward_ragged": lambda args: (
            _write_images(args[3], [args[6] * 3 * h * w for h, w in zip(args[4], args[5])]), _write_losses(args[24])),
        "esacb200_reproj_loss_ragged": lambda args: (
            _write_images(args[3], [3 * h * w for h, w in zip(args[4], args[5])]), _write_losses(args[16])),
        "esacb200_coord_loss_ragged": lambda args: (
            _write_images(args[8], [3 * h * w for h, w in zip(args[3], args[4])]), _write_losses(args[10])),
        "esacb200_hypotheses_backward_ragged": lambda args: (
            _write_images(args[4], [args[7] * 3 * h * w for h, w in zip(args[5], args[6])])),
    }
    return ctx


def _leaves(coords, form):
    if form == "list":
        return [c.clone().requires_grad_(True) for c in coords.unbind(0)]
    return coords.clone().requires_grad_(True)


def _grads(x):
    return [g for g in x.grad.unbind(0)] if torch.is_tensor(x) else [c.grad for c in x]


@pytest.mark.parametrize("op", ["esac_loss_batch", "reproj_loss", "coord_loss", "esac_hypotheses_batch"])
def test_autograd_nodes_give_the_same_gradients_stacked_and_listed(filled, batch, op):
    coords, assign, gts, pred = batch["coords"], batch["assign"], batch["gts"], batch["pred"]
    w = torch.tensor([0.5, -2.0, 3.0])
    got = []
    for form in ("stacked", "list"):
        if op == "esac_loss_batch":
            x = _leaves(coords, form)
            lp = torch.zeros(B, E, requires_grad=True)
            losses = autograd.esac_loss_batch(x, lp, assign, gts, 1.0, 100.0, 100.0, *CAMS, *TAIL)
            assert losses.tolist() == [1.0, 2.0, 3.0]
            (losses * w).sum().backward()
            scale, like = w, coords
            assert torch.equal(lp.grad, autograd._gating_rows([1.0, 2.0, 3.0], assign, E, False) * w[:, None])
        elif op == "esac_hypotheses_batch":
            x = _leaves(coords, form)
            scores, poses, _ = autograd.esac_hypotheses_batch(x, assign, *CAMS, *TAIL)
            scores.sum().backward()
            scale, like = torch.ones(B), coords
        else:
            x = _leaves(pred, form)
            fn = autograd.reproj_loss if op == "reproj_loss" else autograd.coord_loss
            gt = batch["gt_coords"] if form == "stacked" else list(batch["gt_coords"].unbind(0))
            loss = fn(x, gts, 525.0, 0, 0, 10.0) if op == "reproj_loss" else fn(x, gt, 10.0)
            assert loss.item() == 2.0
            (3.0 * loss).backward()
            scale, like = torch.full((B,), 3.0 / B), pred
        got.append(_grads(x))
        for g, e in zip(got[-1], _expected(like, scale)):
            assert torch.equal(g, e), (op, form)
    for a, b in zip(*got):
        assert torch.equal(a, b)
