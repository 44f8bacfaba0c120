"""api.backward_async / api.reserve_backward_async / autograd.esac_loss_async without a GPU: argument errors raised before
any context exists (the tensors here are CPU tensors; the dtype and shape checks come before the device check), the
refinement group rule the host and the stream-ordered backward's kernel share, and the rounding of the gating gradient."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.autograd import _gating_grad, esac_loss_async

LOSS = (1.0, 100.0, 100.0)              # wLossRot, wLossTrans, lossCut
TAIL = (10.0, 100.0, 0.5, 100.0, 8)     # tau, alpha, beta, maxReproj, sub
GOLDEN = Path(__file__).resolve().parent / "golden" / "pick_group_parent.json"


def _args(B=2, E=3, H=6, W=8, M=16):
    lead = (B,) if B else ()
    return dict(sceneCoordinates=torch.zeros(lead + (E, 3, H, W)), outGradients=torch.zeros(lead + (E, 3, H, W)),
                hypAssignment=torch.zeros(lead + (M,), dtype=torch.int64), gtPoses=torch.eye(4).expand(lead + (4, 4)).clone(),
                shifts=torch.zeros(lead + (2,), dtype=torch.int32), cameras=torch.ones(lead + (3,)),
                outLosses=torch.zeros(lead, dtype=torch.float64), outStatus=torch.zeros(lead, dtype=torch.int32))


def _call(**kw):
    a = _args(**{k: kw.pop(k) for k in ("B", "E", "H", "W", "M") if k in kw})
    a.update(kw)
    api.backward_async(a["sceneCoordinates"], a["outGradients"], a["hypAssignment"], a["gtPoses"], a["shifts"], a["cameras"],
                       *LOSS, *TAIL, a["outLosses"], a["outStatus"])


@pytest.mark.parametrize("B", [0, 2])
def test_cpu_tensors_are_refused_after_the_shape_checks(B):
    with pytest.raises(RuntimeError, match=r"backward_async takes CUDA tensors only \(sceneCoordinates is on the CPU\)"):
        _call(B=B)


def test_numpy_arrays_are_refused():
    with pytest.raises(RuntimeError, match=r"backward_async takes torch CUDA tensors only \(sceneCoordinates"):
        _call(sceneCoordinates=np.zeros((2, 3, 3, 6, 8), np.float32))
    with pytest.raises(RuntimeError, match=r"backward_async takes torch CUDA tensors only \(outGradients"):
        _call(outGradients=np.zeros((2, 3, 3, 6, 8), np.float32))
    with pytest.raises(RuntimeError, match=r"backward_async takes torch CUDA tensors only \(outLosses"):
        _call(outLosses=np.zeros(2))


@pytest.mark.parametrize("name,value,msg", [
    ("sceneCoordinates", torch.zeros(2, 3, 3, 6, 8, dtype=torch.float64), "expected scalar type Float but found Double"),
    ("outGradients", torch.zeros(2, 3, 3, 6, 8, dtype=torch.float64), r"Float but found Double \(outGradients\)"),
    ("hypAssignment", torch.zeros(2, 16, dtype=torch.int32), "expected scalar type Long but found Int"),
    ("gtPoses", torch.zeros(2, 4, 4, dtype=torch.float64), r"Float but found Double \(gtPoses\)"),
    ("shifts", torch.zeros(2, 2, dtype=torch.int64), r"expected scalar type Int but found Long \(shifts\)"),
    ("cameras", torch.zeros(2, 3, dtype=torch.float64), r"expected scalar type Float but found Double \(cameras\)"),
    ("outLosses", torch.zeros(2, dtype=torch.float32), r"expected scalar type Double but found Float \(outLosses\)"),
    ("outStatus", torch.zeros(2, dtype=torch.int64), r"expected scalar type Int but found Long \(outStatus\)"),
    ("gtPoses", torch.zeros(4, 4), r"expected 3 dims but tensor has 2 \(gtPoses\)"),
    ("outGradients", torch.zeros(3, 3, 6, 8), r"expected 5 dims but tensor has 4 \(outGradients\)"),
    ("hypAssignment", torch.zeros(16, dtype=torch.int64), r"expected 2 dims but tensor has 1 \(hypAssignment\)"),
])
def test_dtype_and_rank(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _call(**{name: value})


@pytest.mark.parametrize("name,value,msg", [
    ("hypAssignment", torch.zeros(3, 16, dtype=torch.int64), r"hypAssignment must be \[2, 16\] for 2 image"),
    ("shifts", torch.zeros(3, 2, dtype=torch.int32), r"shifts must be \[2, 2\]"),
    ("cameras", torch.zeros(1, 3), r"cameras must be \[2, 3\]"),
    ("outGradients", torch.zeros(2, 3, 3, 6, 9), r"outGradients must be a contiguous \[2, 3, 3, 6, 8\]"),
    ("outGradients", torch.zeros(2, 3, 3, 8, 6).transpose(3, 4), r"outGradients must be a contiguous"),
    ("gtPoses", torch.zeros(3, 4, 4), r"gtPoses must be a contiguous \[2, 4, 4\]"),
    ("gtPoses", torch.zeros(2, 4, 4).transpose(1, 2), r"gtPoses must be a contiguous"),
    ("outLosses", torch.zeros(3, dtype=torch.float64), r"outLosses must be a contiguous \[2\]"),
    ("outStatus", torch.zeros(4, dtype=torch.int32)[::2], r"outStatus must be a contiguous \[2\]"),
    ("sceneCoordinates", torch.zeros(2, 3, 4, 6, 8), r"must be \[B,E,3,H,W\]"),
    ("sceneCoordinates", torch.zeros(2, 3, 3, 8, 6).transpose(3, 4), "sceneCoordinates must be contiguous"),
    ("hypAssignment", torch.zeros(1, 16, dtype=torch.int64).expand(2, 16), "rows back to back"),
])
def test_shapes_and_layouts(name, value, msg):
    with pytest.raises(RuntimeError, match=msg):
        _call(**{name: value})


def test_batch_size_mismatches():
    with pytest.raises(RuntimeError, match=r"outGradients must be a contiguous \[2, 3, 3, 6, 8\]"):
        _call(outGradients=torch.zeros(3, 3, 3, 6, 8))
    with pytest.raises(RuntimeError, match=r"outStatus must be a contiguous \[2\]"):
        _call(outStatus=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(RuntimeError, match=r"expected 1 dims but tensor has 0 \(outLosses\)"):
        _call(outLosses=torch.zeros((), dtype=torch.float64))


def test_sizes():
    with pytest.raises(RuntimeError, match="too small to draw 4 distinct cells"):
        _call(H=2, W=3)
    with pytest.raises(RuntimeError, match="no hypothesis"):
        _call(M=0)
    with pytest.raises(RuntimeError, match="no image or no expert"):
        _call(B=2, E=0)


def test_one_image_takes_unbatched_tensors():
    with pytest.raises(RuntimeError, match="backward_async takes CUDA tensors only"):
        _call(B=0)
    with pytest.raises(RuntimeError, match=r"expected 0 dims but tensor has 1 \(outLosses\)"):
        _call(B=0, outLosses=torch.zeros(1, dtype=torch.float64))
    with pytest.raises(RuntimeError, match=r"gtPoses must be a contiguous \[4, 4\]"):
        _call(B=0, gtPoses=torch.zeros(4, 4).t())


@pytest.mark.parametrize("sizes", [(0, 1, 6, 8, 16), (1, 1, 6, 8, 0), (1, -1, 6, 8, 16), (1, 1, 0, 8, 16)])
def test_reserve_sizes(sizes):
    with pytest.raises(RuntimeError, match="reserve_backward_async: sizes must be positive"):
        api.reserve_backward_async(*sizes)


def test_esac_loss_async_refuses_cpu_tensors():
    a = _args(B=2)
    with pytest.raises(RuntimeError, match="backward_async takes CUDA tensors only"):
        esac_loss_async(a["sceneCoordinates"], torch.zeros(2, 3), a["hypAssignment"], a["gtPoses"], a["shifts"], a["cameras"],
                        *LOSS, *TAIL)


def test_pick_group_rule_reproduces_the_host_table(lib):
    """refine_group_rule, which the host's pick_group and the stream-ordered backward's refinement kernel both evaluate,
    against the groups pick_group chose before the rule was shared (golden/pick_group_parent.json, run-length encoded per
    "N coresident refine_group refine_jobs_per_group" over job counts 1..1024)."""
    table = json.loads(GOLDEN.read_text())
    assert len(table) == 108
    fn = lib.esacb200_host_pick_group
    fn.argtypes = [C.c_int] * 5
    fn.restype = C.c_int
    for key, runs in table.items():
        N, cores, opt, jpg = (int(v) for v in key.split())
        want = [g for g, n in runs for _ in range(n)]
        assert len(want) == 1024
        got = [fn(N, cores, opt, jpg, n) for n in range(1, 1025)]
        assert got == want, key


def test_gating_gradient_rounds_as_esac_loss():
    """esac_loss builds the gating gradient as `loss * torch.histc(...)` with loss a Python float: a float32 product of the
    float32-rounded loss.  _gating_grad (device-side, no .cpu()) must give the same bits; a float64 product would not."""
    rng = np.random.default_rng(7)
    differs_in_float64 = 0
    for _ in range(400):
        B, E, M = int(rng.integers(1, 4)), int(rng.integers(1, 30)), int(rng.integers(1, 600))
        losses = torch.from_numpy(rng.random(B) * 10.0 ** rng.uniform(-5, 4, B))
        assign = torch.from_numpy(rng.integers(0, E, (B, M)))
        want = torch.stack([float(losses[b]) * torch.histc(assign[b].float(), bins=E, min=0, max=E - 1) for b in range(B)])
        assert torch.equal(_gating_grad(losses, assign, E, False), want)
        sel = torch.zeros(B, E)
        for b in range(B):
            sel[b, int(assign[b, 0])] = float(losses[b])
        assert torch.equal(_gating_grad(losses, assign, E, True), sel)
        hist = torch.stack([torch.histc(assign[b].float(), bins=E, min=0, max=E - 1) for b in range(B)])
        differs_in_float64 += not torch.equal((losses[:, None] * hist.double()).float(), want)
    assert differs_in_float64 > 0


def test_gating_gradient_ignores_bad_indices():
    losses = torch.tensor([2.5, 1.0], dtype=torch.float64)
    assign = torch.tensor([[0, 1, 1, 3], [2, 2, 0, 1]])   # 3 is outside [0, 3)
    g = _gating_grad(losses, assign, 3, False)
    assert g.tolist() == [[2.5, 5.0, 0.0], [1.0, 1.0, 2.0]]
