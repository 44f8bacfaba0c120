"""Run only the experts that draw hypotheses in a captured CUDA graph, as the reference's loops do.

test_esac.py:179-185 and train_esac.py:143-145 run expert e only `if count > 0`, and ensemble.update
(expert_ensemble.py:58-68) steps only those experts.  A captured graph is a fixed sequence of kernels, so without a gate a
replay runs, and trains, every expert.  An ExpertGate turns each `run(e, fn)` of a capture into a conditional node of the
graph: a kernel that reads the hypothesis histogram on the device decides, at every replay, which of them run.

    gate = ExpertGate(E)
    def step():
        ...draw e_hyps and hist on the device (api.assign_hypotheses_async)...
        gate.arm(hist)
        for e in range(E):
            gate.run(e, lambda e=e: prediction[e].copy_(experts[e](image)[0]))
        ...
    step()                                    # eager: reads hist once, runs the active experts
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        step()                                # captured: every region is marked
    gate.finalize(graph)                      # the regions become conditional nodes; the graph is instantiated
    graph.replay()

The same step function serves the eager warm-up and the capture.  A gate belongs to one graph; the work of a region runs
on the capturing stream (a stream forked inside it must join before it ends), and conditional nodes need a CUDA 12.3
driver.  n is generic: index b * E + e gates expert e of image b of a batch.
"""
from __future__ import annotations

import ctypes as C

from . import api


def _capturing() -> bool:
    import torch
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


class ExpertGate:
    """n regions' switches: region i of a captured step runs at replay only where counts[i] > 0 (see the module)."""

    def __init__(self, n: int, device=None):
        if isinstance(n, bool) or not isinstance(n, int):
            raise RuntimeError(f"ExpertGate: n must be an int, got {type(n).__name__}")
        if not 1 <= n <= api.MAX_EXPERTS:
            raise RuntimeError(f"ExpertGate: n={n} outside [1, {api.MAX_EXPERTS}]")
        import torch
        self.n = n
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"ExpertGate: device must be a CUDA device, got {self.device}")
        self._ctx = api.context(self.device.index if self.device.index is not None else torch.cuda.current_device())
        h = C.c_void_p()
        self._ctx.check(self._ctx.lib.esacb200_gate_create(self._ctx.handle, n, C.byref(h)))
        self._handle = h
        self._active = None   # eager: which regions run, read from the last arm()

    def close(self):
        if getattr(self, "_handle", None):
            self._ctx.lib.esacb200_gate_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> int:
        import torch
        return torch.cuda.current_stream(self.device).cuda_stream

    def arm(self, counts):
        """counts: float32 CUDA tensor of n elements ([n], or [B,E] with B * E = n), e.g. the histogram of
        assign_hypotheses_async.  While capturing, the graph reads it on the device; eagerly, it is read to the host once
        (the reference's .cpu() of the histogram)."""
        import torch
        if not isinstance(counts, torch.Tensor):
            raise RuntimeError(f"ExpertGate.arm: counts must be a torch tensor, got {type(counts).__name__}")
        if counts.dtype != torch.float32:
            raise RuntimeError(f"ExpertGate.arm: expected scalar type Float but found {api._dtype_name(counts)} (counts)")
        if counts.dim() not in (1, 2):
            raise RuntimeError(f"ExpertGate.arm: counts must be [n] or [B,E], got {list(counts.shape)}")
        if int(counts.numel()) != self.n:
            raise RuntimeError(f"ExpertGate.arm: counts holds {int(counts.numel())} elements, the gate {self.n}")
        if not counts.is_cuda or counts.device != self.device:
            raise RuntimeError(f"ExpertGate.arm: counts must live on {self.device}, got {counts.device}")
        if not counts.is_contiguous():
            raise RuntimeError("ExpertGate.arm: counts must be contiguous (a copy would not be captured with the call)")
        if _capturing():
            self._ctx.check(self._ctx.lib.esacb200_gate_arm(self._handle, counts.data_ptr(), self._stream()))
        else:
            self._active = (counts.reshape(-1) > 0).tolist()

    def _mark(self, i: int, begin: bool):
        self._ctx.check(self._ctx.lib.esacb200_gate_mark(self._handle, i, int(begin), self._stream()))

    def run(self, i: int, fn):
        """Region i: while capturing, fn() between a begin and an end marker; eagerly, fn() only if counts[i] > 0 at the
        last arm().  Returns what fn returns (None where it did not run)."""
        if isinstance(i, bool) or not isinstance(i, int) or not 0 <= i < self.n:
            raise RuntimeError(f"ExpertGate.run: index {i!r} outside [0, {self.n})")
        if _capturing():
            self._mark(i, True)
            out = fn()
            self._mark(i, False)
            return out
        if self._active is None:
            raise RuntimeError("ExpertGate.run: arm() the gate before running its regions eagerly")
        return fn() if self._active[i] else None

    def finalize(self, graph):
        """Rewrites a captured torch.cuda.CUDAGraph(keep_graph=True): each region becomes a conditional node on its
        switch; then instantiates the graph.  Raises RuntimeError with the library's reason (the graph is then left as
        captured) or if the graph was not built with keep_graph=True."""
        import torch
        if not isinstance(graph, torch.cuda.CUDAGraph):
            raise RuntimeError(f"ExpertGate.finalize takes a torch.cuda.CUDAGraph, got {type(graph).__name__}")
        try:
            raw = graph.raw_cuda_graph()
        except RuntimeError as e:
            raise RuntimeError("ExpertGate.finalize needs a graph captured with torch.cuda.CUDAGraph(keep_graph=True) "
                               f"and not yet reset ({e})") from None
        if not raw:
            raise RuntimeError("ExpertGate.finalize needs a graph captured with torch.cuda.CUDAGraph(keep_graph=True)")
        self._ctx.check(self._ctx.lib.esacb200_gate_finalize(self._handle, raw))
        graph.instantiate()
