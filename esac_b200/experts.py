"""Inference of a stack of the reference's experts (code/expert.py: Expert) on the tensor cores.

ExpertStack takes the experts' own state dicts (`torch.load('esac_<sid>.net')[1:]`, the list ExpertEnsemble.save writes
behind the gating network's) and predicts the scene coordinates of the (image, expert) pairs that draw hypotheses, every
layer of all of them in one launch (include/esac_b200.h: esacb200_experts_*).  The numerics are TF32 operands with fp32
accumulation and fp32 activations, the regime of the reference's convolutions under torch's default
`torch.backends.cudnn.allow_tf32 = True`; expert e's output for image b does not depend on the other pairs of the call.

    stack = ExpertStack(torch.load('esac_scene.net')[1:], 'cuda')
    prediction = stack.forward(image, hist)          # [B,E,3,ceil(H/8),ceil(W/8)], zero planes where hist is 0

forward_async writes into a caller-owned buffer on torch's current stream without a host synchronisation, so a CUDA graph
can capture it; reserve(B, H, W) sizes the workspace before the capture.
"""
from __future__ import annotations

import ctypes as C

from . import api
from .compat import OUTPUT_SUBSAMPLE
# Expert.__init__'s layers in state-dict order: name, Cin, Cout, kernel size, stride (padding k // 2).
LAYERS = (("conv1", 3, 32, 3, 1), ("conv2", 32, 64, 3, 2), ("conv3", 64, 128, 3, 2), ("conv4", 128, 256, 3, 2),
          ("res1_conv1", 256, 256, 3, 1), ("res1_conv2", 256, 256, 1, 1), ("res1_conv3", 256, 256, 3, 1),
          ("res2_conv1", 256, 512, 3, 1), ("res2_conv2", 512, 512, 1, 1), ("res2_conv3", 512, 512, 3, 1),
          ("res2_skip", 256, 512, 1, 1),
          ("res3_conv1", 512, 512, 1, 1), ("res3_conv2", 512, 512, 1, 1), ("res3_conv3", 512, 512, 1, 1),
          ("fc1", 512, 512, 1, 1), ("fc2", 512, 512, 1, 1), ("fc3", 512, 3, 1, 1))


def state_dict_shapes() -> dict:
    """Key -> shape of one expert's state dict, in the order the C ABI takes the tensors."""
    shapes = {}
    for name, cin, cout, k, _ in LAYERS:
        shapes[name + ".weight"] = (cout, cin, k, k)
        shapes[name + ".bias"] = (cout,)
    shapes["mean"] = (3,)
    return shapes


def prediction_size(H: int, W: int) -> tuple:
    return -(-H // OUTPUT_SUBSAMPLE), -(-W // OUTPUT_SUBSAMPLE)


def _check_state_dict(who: str, sd, want: dict, cls: str) -> list:
    """The tensors of `who`'s state dict in ABI order, as contiguous float32: exactly the keys of a `cls` state dict with
    the shapes `want` (key -> shape, in ABI order)."""
    import torch
    have = set(sd.keys())
    missing, extra = [k for k in want if k not in have], sorted(have - set(want))
    if missing or extra:
        raise RuntimeError(f"{who}: state dict keys differ from {cls}'s (missing {missing}, unexpected {extra})")
    out = []
    for k, shape in want.items():
        t = sd[k]
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise RuntimeError(f"{who}: {k} must be a floating-point tensor, got "
                               f"{t.dtype if isinstance(t, torch.Tensor) else type(t).__name__}")
        if tuple(t.shape) != shape:
            raise RuntimeError(f"{who}: {k} must be {list(shape)}, got {list(t.shape)}")
        out.append(t.detach().to(torch.float32).contiguous())
    return out


class ExpertStack:
    """E experts, packed once on `device` as [expert][Cout][kh][kw][Cin] per layer, TF32-rounded where the tensor cores
    read them."""

    def __init__(self, state_dicts, device="cuda"):
        import torch
        state_dicts = list(state_dicts)
        E = len(state_dicts)
        if not 1 <= E <= api.MAX_EXPERTS:
            raise RuntimeError(f"ExpertStack: {E} experts, outside [1, {api.MAX_EXPERTS}]")
        tensors = [t for i, sd in enumerate(state_dicts)
                   for t in _check_state_dict(f"expert {i}", sd, state_dict_shapes(), "Expert")]
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"ExpertStack runs on a CUDA device, not {self.device}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.E = E
        lib = api.load_library()
        self.packed = torch.empty(int(lib.esacb200_experts_packed_floats(E)), dtype=torch.float32, device=self.device)
        ptrs = (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        with torch.cuda.device(self.device):
            ctx = api._pick_ctx(self.device.index)
            ctx.check(lib.esacb200_experts_pack(ctx.handle, E, ptrs, self.packed.data_ptr()))
        self.workspace = None
        self.frozen = False   # a captured graph holds the workspace: it is never freed or replaced from then on

    def workspace_bytes(self, B: int, H: int, W: int) -> int:
        n = int(api.load_library().esacb200_experts_workspace_bytes(int(B), self.E, int(H), int(W)))
        if n < 0:
            raise RuntimeError(f"ExpertStack: B={B} E={self.E} H={H} W={W}: sizes outside the supported range "
                               "(B * E <= 65535, sides <= 8192)")
        return n

    def reserve(self, B: int, H: int, W: int):
        """Sizes the workspace for B images of HxW (call it before capturing forward_async in a graph)."""
        import torch
        if min(int(B), int(H), int(W)) < 1:
            raise RuntimeError(f"ExpertStack.reserve: sizes must be positive, got B={B} H={H} W={W}")
        n = self.workspace_bytes(B, H, W)
        if self.workspace is None or self.workspace.numel() < n:
            if self.frozen:
                raise RuntimeError(f"ExpertStack.reserve: B={B} at {H}x{W} needs {n} workspace bytes, more than the "
                                   f"{self.workspace.numel()} a captured graph already uses (reserve the largest shape "
                                   "before the first capture)")
            self.workspace = None
            self.workspace = torch.empty(n, dtype=torch.uint8, device=self.device)

    def forward_async(self, image, hist, out):
        """Predictions of the active pairs into out float32 [B,E,3,ceil(H/8),ceil(W/8)] on torch's current stream, with no
        host synchronisation.  image: float32 [B,3,H,W], or [1,3,H,W] for every image of the batch; hist: float32 [B,E]
        (pair (b, e) runs when hist[b,e] > 0; assign_hypotheses_async's outHist) or None (all pairs run).  Outside a capture
        the workspace grows as needed; inside one it must have been reserved, and once a capture has used it, it no longer
        grows: a later call that needs more raises."""
        import torch
        call = "ExpertStack.forward_async"
        if not api._is_torch(image):
            raise RuntimeError(f"{call} takes torch CUDA tensors only (image is a {type(image).__name__})")
        api._check(image, "Float", 4, "image")
        if int(image.shape[1]) != 3:
            raise RuntimeError(f"image must be [B,3,H,W], got {list(image.shape)}")
        if not api._is_torch(out):
            raise RuntimeError(f"{call} takes torch CUDA tensors only (out is a {type(out).__name__})")
        api._check(out, "Float", 5, "out")
        B, H, W = int(out.shape[0]), int(image.shape[2]), int(image.shape[3])
        if int(image.shape[0]) not in (1, B):
            raise RuntimeError(f"image holds {int(image.shape[0])} images for out's batch of {B} (need 1 or {B})")
        fixed = {"out": (out, "Float", (B, self.E, 3) + prediction_size(H, W))}
        if hist is not None:
            fixed["hist"] = (hist, "Float", (B, self.E))

        def check():
            if not image.is_contiguous():
                raise RuntimeError("image must be contiguous (a copy would not be captured with the call)")
        ctx = api._async_context(call, fixed, [("image", image)], check)
        if image.device != self.device:
            raise RuntimeError(f"{call}: tensors on {image.device}, the experts on {self.device}")
        need = self.workspace_bytes(B, H, W)
        capturing = torch.cuda.is_current_stream_capturing()
        if (self.workspace is None or self.workspace.numel() < need) and not capturing:
            self.reserve(B, H, W)
        ws = self.workspace
        self.frozen = self.frozen or (capturing and ws is not None)
        ctx.check(ctx.lib.esacb200_experts_forward_async(
            ctx.handle, B, self.E, H, W, image.data_ptr(), int(image.shape[0]),
            hist.data_ptr() if hist is not None else None, self.packed.data_ptr(),
            ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0, out.data_ptr()))

    def forward(self, image, hist=None):
        """The predictions as a new tensor [B,E,3,ceil(H/8),ceil(W/8)] (B from hist, else from image)."""
        import torch
        B = int(hist.shape[0]) if hist is not None and api._is_torch(hist) and hist.dim() == 2 else int(image.shape[0])
        h, w = prediction_size(int(image.shape[2]), int(image.shape[3])) if api._is_torch(image) and image.dim() == 4 else (1, 1)
        out = torch.empty((B, self.E, 3, h, w), dtype=torch.float32,
                          device=image.device if api._is_torch(image) and image.is_cuda else self.device)
        self.forward_async(image, hist, out)
        return out
