"""Argument errors of the expert gate (esac_b200.gate.ExpertGate, esacb200_gate_*) and of api.assign_hypotheses_async: the
C entries refuse null handles, and the Python checks raise before any context exists, so all of this runs without a GPU
(the tensors here are CPU tensors; the dtype and shape checks come before the device check)."""
import ctypes as C

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.gate import ExpertGate


def test_c_entries_refuse_null_handles(lib):
    ERR_ARG = -2
    h = C.c_void_p()
    assert lib.esacb200_gate_create(None, 4, C.byref(h)) == ERR_ARG and not h.value
    assert lib.esacb200_gate_arm(None, None, None) == ERR_ARG
    assert lib.esacb200_gate_mark(None, 0, 1, None) == ERR_ARG
    assert lib.esacb200_gate_finalize(None, None) == ERR_ARG
    lib.esacb200_gate_destroy(None)  # a no-op, like free(NULL)
    assert lib.esacb200_assign_hypotheses_async(None, 1, 4, 8, None, -1, 0, None, None, None, None) == ERR_ARG


@pytest.mark.parametrize("n, match", [(0, r"n=0 outside \[1, 1024\]"), (1025, r"n=1025 outside \[1, 1024\]"),
                                      (-3, r"n=-3 outside"), (2.0, "n must be an int"), (True, "n must be an int")])
def test_gate_size_is_checked_before_any_context(n, match):
    with pytest.raises(RuntimeError, match=match):
        ExpertGate(n)
    assert not api._contexts


def _unbuilt_gate(n):
    """An ExpertGate whose library handle was never created: arm() and run() check their arguments before they use it."""
    g = ExpertGate.__new__(ExpertGate)
    g.n, g.device, g._active, g._handle = n, torch.device("cuda", 0), None, None
    return g


def test_arm_checks_counts_before_any_context():
    g = _unbuilt_gate(6)
    with pytest.raises(RuntimeError, match="counts must be a torch tensor"):
        g.arm(np.ones(6, np.float32))
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        g.arm(torch.ones(6, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Long"):
        g.arm(torch.ones(6, dtype=torch.int64))
    with pytest.raises(RuntimeError, match=r"counts must be \[n\] or \[B,E\], got \[1, 2, 3\]"):
        g.arm(torch.ones(1, 2, 3))
    with pytest.raises(RuntimeError, match=r"counts must be \[n\] or \[B,E\], got \[\]"):
        g.arm(torch.ones(()))
    with pytest.raises(RuntimeError, match="counts holds 5 elements, the gate 6"):
        g.arm(torch.ones(5))
    with pytest.raises(RuntimeError, match="counts holds 8 elements, the gate 6"):
        g.arm(torch.ones(2, 4))
    with pytest.raises(RuntimeError, match="counts must live on cuda:0, got cpu"):
        g.arm(torch.ones(2, 3))   # [B, E] with B * E = n passes the shape checks
    assert not api._contexts


def test_run_checks_its_index_and_needs_an_arm_eagerly():
    g = _unbuilt_gate(3)
    for bad in (-1, 3, 1.0, True):
        with pytest.raises(RuntimeError, match=r"outside \[0, 3\)"):
            g.run(bad, lambda: None)
    with pytest.raises(RuntimeError, match=r"arm\(\) the gate before running its regions eagerly"):
        g.run(0, lambda: None)
    g._active = [True, False, True]   # what an eager arm() of counts [2, 0, 0.5] leaves
    ran = []
    assert [g.run(i, lambda i=i: ran.append(i) or i) for i in range(3)] == [0, None, 2] and ran == [0, 2]


def test_finalize_needs_a_torch_graph():
    g = _unbuilt_gate(2)
    with pytest.raises(RuntimeError, match="takes a torch.cuda.CUDAGraph, got int"):
        g.finalize(0)


def _assign_args(B=2, E=4, M=8):
    lead = (B,) if B else ()
    return dict(gatingProbs=torch.ones(lead + (E,)), hypotheses=M, seed=torch.zeros(1, dtype=torch.int64),
                outAssign=torch.zeros(lead + (M,), dtype=torch.int64), outHist=torch.zeros(lead + (E,)),
                outStatus=torch.zeros(lead, dtype=torch.int32))


def _assign(**kw):
    a = _assign_args(**{k: kw.pop(k) for k in ("B", "E", "M") if k in kw})
    a.update(kw)
    api.assign_hypotheses_async(a["gatingProbs"], a["hypotheses"], a["seed"], a["outAssign"], a["outHist"], a["outStatus"],
                                maxExperts=2)


def test_assign_async_checks_before_any_context():
    with pytest.raises(RuntimeError, match=r"torch CUDA tensors only \(gatingProbs is a ndarray\)"):
        _assign(gatingProbs=np.ones((2, 4), np.float32))
    with pytest.raises(RuntimeError, match="expected scalar type Float but found Double"):
        _assign(gatingProbs=torch.ones(2, 4, dtype=torch.float64))
    with pytest.raises(RuntimeError, match=r"gatingProbs must be \[B,E\] or \[E\], got \[1, 2, 4\]"):
        _assign(gatingProbs=torch.ones(1, 2, 4))
    with pytest.raises(RuntimeError, match="sizes must be positive, got B=2 E=4 M=0"):
        _assign(hypotheses=0)
    with pytest.raises(RuntimeError, match="E=1025 exceeds the 1024 experts one CTA holds"):
        _assign(E=1025)
    with pytest.raises(RuntimeError, match=r"seed must be an int64 CUDA tensor of one element, got Int\[1\]"):
        _assign(seed=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(RuntimeError, match=r"seed must be an int64 CUDA tensor of one element, got Long\[2\]"):
        _assign(seed=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="seed must be an int64 CUDA tensor of one element, got int"):
        _assign(seed=7)
    with pytest.raises(RuntimeError, match="expected scalar type Long but found Int \\(outAssign\\)"):
        _assign(outAssign=torch.zeros(2, 8, dtype=torch.int32))
    with pytest.raises(RuntimeError, match=r"outAssign must be a contiguous \[2, 8\] tensor, got \[2, 9\]"):
        _assign(outAssign=torch.zeros(2, 9, dtype=torch.int64))
    with pytest.raises(RuntimeError, match=r"expected 2 dims but tensor has 1 \(outHist\)"):
        _assign(outHist=torch.zeros(4))
    with pytest.raises(RuntimeError, match=r"outHist must be a contiguous \[2, 4\] tensor, got \[2, 5\]"):
        _assign(outHist=torch.zeros(2, 5))
    with pytest.raises(RuntimeError, match=r"outStatus must be a contiguous \[2\] tensor, got \[1\]"):
        _assign(outStatus=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="gatingProbs must be contiguous"):
        _assign(gatingProbs=torch.ones(4, 2).t())
    with pytest.raises(RuntimeError, match=r"assign_hypotheses_async takes CUDA tensors only \(gatingProbs is on the CPU\)"):
        _assign()
    with pytest.raises(RuntimeError, match=r"CUDA tensors only \(gatingProbs is on the CPU\)"):
        _assign(B=0, outHist=None)   # one image: [E] probabilities, [M] assignment, [] status
    assert not api._contexts
