"""Inference of the reference's gating network (code/gating.py: Gating) on the device.

GatingNet takes the network's state dict (`torch.load('esac_<sid>.net')[0]`, the first entry ExpertEnsemble.save writes,
or `torch.load('gating_<sid>.net')`) and reads the expert count E and the capacity (1 for room environments, 2 for clustered
ones) from its shapes.  Its forward is Gating.forward: log-probabilities [B,E] over the experts, in one launch per stage
(include/esac_b200.h: esacb200_gating_*).  The numerics are the expert stack's: TF32 operands with fp32 accumulation where
the tensor cores run (conv4 and res1_conv1..3), fp32 elsewhere.  Image b's output is bitwise independent of the batch, of
its place in it and of the run: no split-K, no atomics.

    gating = GatingNet(torch.load('esac_scene.net')[0], 'cuda')
    log_p = gating.forward(image)                       # [B,E], like Gating.forward(image)

forward_async writes into caller-owned buffers on torch's current stream without a host synchronisation, so a CUDA graph
can capture it, and can write exp(log_p) as well, the probabilities assign_hypotheses_async draws from; reserve(B, H, W)
sizes the workspace before the capture.
"""
from __future__ import annotations

import ctypes as C

from . import api
from .experts import _check_state_dict


def layers(E: int, capacity: int) -> tuple:
    """Gating.__init__'s layers in state-dict order: name, Cin, Cout, kernel size, stride (padding k // 2)."""
    c, cc = 64 * capacity, 64 * capacity * capacity
    return (("conv1", 3, 8, 3, 1), ("conv2", 8, 16, 3, 2), ("conv3", 16, 32, 3, 2), ("conv4", 32, c, 3, 2),
            ("res1_conv1", c, c, 3, 1), ("res1_conv2", c, c, 1, 1), ("res1_conv3", c, c, 3, 1),
            ("fc1", c, cc, 1, 1), ("fc2", cc, cc, 1, 1), ("fc3", cc, E, 1, 1))


def state_dict_shapes(E: int, capacity: int) -> dict:
    """Key -> shape of the state dict of Gating(E, capacity), in the order the C ABI takes the tensors."""
    shapes = {}
    for name, cin, cout, k, _ in layers(E, capacity):
        shapes[name + ".weight"] = (cout, cin, k, k)
        shapes[name + ".bias"] = (cout,)
    return shapes


def network_size(sd) -> tuple:
    """(E, capacity) of a Gating state dict, from fc3's and conv4's weights."""
    import torch
    for key in ("fc3.weight", "conv4.weight"):
        if key not in sd:
            raise RuntimeError(f"gating: state dict keys differ from Gating's (missing ['{key}'])")
        if not isinstance(sd[key], torch.Tensor) or sd[key].dim() != 4:
            raise RuntimeError(f"gating: {key} must be a 4-d floating-point tensor")
    E, c = int(sd["fc3.weight"].shape[0]), int(sd["conv4.weight"].shape[0])
    if c not in (64, 128):
        raise RuntimeError(f"gating: conv4.weight must be [64, 32, 3, 3] (capacity 1) or [128, 32, 3, 3] (capacity 2), "
                           f"got {list(sd['conv4.weight'].shape)}")
    if not 1 <= E <= api.MAX_EXPERTS:
        raise RuntimeError(f"gating: fc3.weight gives {E} experts, outside [1, {api.MAX_EXPERTS}]")
    return E, c // 64


class GatingNet:
    """Gating(E, capacity), packed once on `device`: conv1 .. conv3 as [k][k][Cin][Cout], conv4 and res1_* as
    [Cout][k][k][Cin] rounded to TF32, fc1 .. fc3 as [Cin][Cout]."""

    def __init__(self, state_dict, device="cuda"):
        import torch
        self.E, self.capacity = network_size(state_dict)
        tensors = _check_state_dict("gating", state_dict, state_dict_shapes(self.E, self.capacity), "Gating")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"GatingNet runs on a CUDA device, not {self.device}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        lib = api.load_library()
        self.packed = torch.empty(int(lib.esacb200_gating_packed_floats(self.E, self.capacity)), dtype=torch.float32,
                                  device=self.device)
        ptrs = (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        with torch.cuda.device(self.device):
            ctx = api._pick_ctx(self.device.index)
            ctx.check(lib.esacb200_gating_pack(ctx.handle, self.E, self.capacity, ptrs, self.packed.data_ptr()))
        self.workspace = None
        self.frozen = False   # a captured graph holds the workspace: it is never freed or replaced from then on

    def workspace_bytes(self, B: int, H: int, W: int) -> int:
        n = int(api.load_library().esacb200_gating_workspace_bytes(int(B), self.E, self.capacity, int(H), int(W)))
        if n < 0:
            raise RuntimeError(f"GatingNet: B={B} H={H} W={W}: sizes outside the supported range "
                               "(B <= 65535, sides <= 8192)")
        return n

    def reserve(self, B: int, H: int, W: int):
        """Sizes the workspace for B images of HxW (call it before capturing forward_async in a graph)."""
        import torch
        if min(int(B), int(H), int(W)) < 1:
            raise RuntimeError(f"GatingNet.reserve: sizes must be positive, got B={B} H={H} W={W}")
        n = self.workspace_bytes(B, H, W)
        if self.workspace is None or self.workspace.numel() < n:
            if self.frozen:
                raise RuntimeError(f"GatingNet.reserve: B={B} at {H}x{W} needs {n} workspace bytes, more than the "
                                   f"{self.workspace.numel()} a captured graph already uses (reserve the largest shape "
                                   "before the first capture)")
            self.workspace = None
            self.workspace = torch.empty(n, dtype=torch.uint8, device=self.device)

    def forward_async(self, image, out_log_probs, out_probs=None):
        """Gating.forward(image) into out_log_probs float32 [B,E], and exp of it into out_probs [B,E] unless None, on
        torch's current stream with no host synchronisation.  image: float32 [B,3,H,W], contiguous.  Outside a capture the
        workspace grows as needed; inside one it must have been reserved, and once a capture has used it, it no longer
        grows: a later call that needs more raises."""
        import torch
        call = "GatingNet.forward_async"
        if not api._is_torch(image):
            raise RuntimeError(f"{call} takes torch CUDA tensors only (image is a {type(image).__name__})")
        api._check(image, "Float", 4, "image")
        if int(image.shape[1]) != 3:
            raise RuntimeError(f"image must be [B,3,H,W], got {list(image.shape)}")
        B, H, W = (int(v) for v in (image.shape[0], image.shape[2], image.shape[3]))
        fixed = {"out_log_probs": (out_log_probs, "Float", (B, self.E))}
        if out_probs is not None:
            fixed["out_probs"] = (out_probs, "Float", (B, self.E))

        def check():
            if not image.is_contiguous():
                raise RuntimeError("image must be contiguous (a copy would not be captured with the call)")
        ctx = api._async_context(call, fixed, [("image", image)], check)
        if image.device != self.device:
            raise RuntimeError(f"{call}: tensors on {image.device}, the network on {self.device}")
        need = self.workspace_bytes(B, H, W)
        capturing = torch.cuda.is_current_stream_capturing()
        if (self.workspace is None or self.workspace.numel() < need) and not capturing:
            self.reserve(B, H, W)
        ws = self.workspace
        self.frozen = self.frozen or (capturing and ws is not None)
        ctx.check(ctx.lib.esacb200_gating_forward_async(
            ctx.handle, B, self.E, self.capacity, H, W, image.data_ptr(), self.packed.data_ptr(),
            ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0, out_log_probs.data_ptr(),
            out_probs.data_ptr() if out_probs is not None else None))

    def forward(self, image):
        """The log-probabilities as a new tensor [B,E], as Gating.forward returns them."""
        import torch
        B = int(image.shape[0]) if api._is_torch(image) and image.dim() == 4 else 1
        out = torch.empty((B, self.E), dtype=torch.float32,
                          device=image.device if api._is_torch(image) and image.is_cuda else self.device)
        self.forward_async(image, out)
        return out
