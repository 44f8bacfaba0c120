"""Oracle for the gating network (esac_b200/gating_net.py, esac_b200/csrc/gating_net.cu).  TEST INFRASTRUCTURE ONLY.

`forward` is the reference's Gating (code/gating.py) written from its layer table as float64 torch.nn.functional calls on
the CPU: conv1 .. conv4 and res1_conv1..3 with ReLU (a plain chain, no residual add), tanh for capacity 1, the mean over
the /8 map, fc1 and fc2 with ReLU, fc3, log_softmax over the experts.  `Gating` restates the reference's module for the
comparisons with torch's own route.  `pack` / `unpack` restate the packed weight layout of include/esac_b200.h in numpy,
with the TF32 rounding (cvt.rna) of the layers the tensor cores read.

Only tests/, tools/ and examples/ may import this module; the product path never does.
"""
from __future__ import annotations

import numpy as np

from esac_b200.gating_net import layers, state_dict_shapes
from oracle.expert_oracle import tf32

ALIGN = 64  # floats: every segment of the packed weights starts on this boundary
FRONT, GEMM = ("conv1", "conv2", "conv3"), ("conv4", "res1_conv1", "res1_conv2", "res1_conv3")


def apply(x, p: dict, capacity: int):
    """Gating.forward on x [B,3,H,W] with parameters p (key -> tensor on x's device and dtype), as functional calls."""
    import torch
    import torch.nn.functional as F
    E = int(p["fc3.weight"].shape[0])
    for name, _, _, k, s in layers(E, capacity):
        x = F.conv2d(x, p[name + ".weight"], p[name + ".bias"], stride=s, padding=k // 2)
        if name != "fc3":
            x = F.relu(x)
        if name == "res1_conv3":
            if capacity == 1:
                x = torch.tanh(x)
            x = x.mean(dim=(2, 3), keepdim=True)
    return F.log_softmax(x, dim=1)[:, :, 0, 0]


def forward(image, sd, capacity: int):
    """Gating.forward of the network with state dict sd on image [B,3,H,W], in float64 on the CPU: [B,E]."""
    import torch
    p = {k: torch.as_tensor(v).detach().to("cpu", torch.float64) for k, v in sd.items()}
    return apply(torch.as_tensor(image).detach().to("cpu", torch.float64), p, capacity)


def make_gating_class():
    """The reference's Gating module (code/gating.py), restated: the same layers, forward and state-dict keys."""
    import torch
    import torch.nn as nn
    import torch.nn.functional as F

    class Gating(nn.Module):
        def __init__(self, num_experts, capacity=1):
            super().__init__()
            self.capacity = capacity
            self.conv1 = nn.Conv2d(3, 8, 3, 1, 1)
            self.conv2 = nn.Conv2d(8, 16, 3, 2, 1)
            self.conv3 = nn.Conv2d(16, 32, 3, 2, 1)
            self.conv4 = nn.Conv2d(32, 64 * capacity, 3, 2, 1)
            self.res1_conv1 = nn.Conv2d(64 * capacity, 64 * capacity, 3, 1, 1)
            self.res1_conv2 = nn.Conv2d(64 * capacity, 64 * capacity, 1, 1, 0)
            self.res1_conv3 = nn.Conv2d(64 * capacity, 64 * capacity, 3, 1, 1)
            self.fc1 = nn.Conv2d(64 * capacity, 64 * capacity ** 2, 1, 1, 0)
            self.fc2 = nn.Conv2d(64 * capacity ** 2, 64 * capacity ** 2, 1, 1, 0)
            self.fc3 = nn.Conv2d(64 * capacity ** 2, num_experts, 1, 1, 0)

        def forward(self, inputs):
            x = inputs
            x = F.relu(self.conv1(x))
            x = F.relu(self.conv2(x))
            x = F.relu(self.conv3(x))
            x = F.relu(self.conv4(x))
            x = F.relu(self.res1_conv1(x))
            x = F.relu(self.res1_conv2(x))
            x = F.relu(self.res1_conv3(x))
            if self.capacity == 1:
                x = torch.tanh(x)
            x = F.avg_pool2d(x, x.size()[2:])
            x = F.relu(self.fc1(x))
            x = F.relu(self.fc2(x))
            x = self.fc3(x)
            x = F.log_softmax(x, dim=1)
            return x[:, :, 0, 0]

    return Gating


def kaiming_state_dict(seed: int, E: int, capacity: int) -> dict:
    """A seeded Kaiming-normal (fan-in, ReLU gain) Gating(E, capacity) with small uniform biases."""
    import torch
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_shapes(E, capacity).items():
        if name.endswith(".weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            sd[name] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        else:
            sd[name] = (torch.rand(shape, generator=g) - 0.5) * 0.1
    return sd


def _round(n: int) -> int:
    return -(-n // ALIGN) * ALIGN


def _segments(E: int, capacity: int):
    """(name, W offset, b offset, (Cout, Cin, k)) per layer, and the total."""
    off, out = 0, []
    for name, cin, cout, k, _ in layers(E, capacity):
        w = off
        off += _round(cout * cin * k * k)
        out.append((name, w, off, (cout, cin, k)))
        off += _round(cout)
    return out, off


def packed_floats(E: int, capacity: int) -> int:
    return _segments(E, capacity)[1]


def _layout(name: str):
    """The permutation of torch's [Cout][Cin][k][k] axes into the packed layout of layer `name`."""
    return (2, 3, 1, 0) if name in FRONT else (0, 2, 3, 1) if name in GEMM else (1, 2, 3, 0)


def pack(sd, capacity: int) -> np.ndarray:
    """The packed float32 weights of the network with state dict sd; zero between segments."""
    E = int(sd["fc3.weight"].shape[0])
    segs, total = _segments(E, capacity)
    out = np.zeros(total, np.float32)
    for name, w_off, b_off, (cout, cin, k) in segs:
        w = np.asarray(sd[name + ".weight"].detach().cpu(), np.float32).transpose(_layout(name)).reshape(-1)
        out[w_off: w_off + w.size] = tf32(w) if name in GEMM else w
        out[b_off: b_off + cout] = np.asarray(sd[name + ".bias"].detach().cpu(), np.float32)
    return out


def unpack(packed: np.ndarray, E: int, capacity: int) -> dict:
    """The state dict (numpy float32, torch's layouts) held by packed weights."""
    segs, _ = _segments(E, capacity)
    sd = {}
    for name, w_off, b_off, (cout, cin, k) in segs:
        perm = _layout(name)
        shape = tuple((cout, cin, k, k)[a] for a in perm)
        w = packed[w_off: w_off + cout * cin * k * k].reshape(shape).transpose(np.argsort(perm))
        sd[name + ".weight"] = np.ascontiguousarray(w)
        sd[name + ".bias"] = packed[b_off: b_off + cout].copy()
    return sd


POOL_CELLS = 128  # cells of the /8 map per pool chunk


def workspace_layout(B: int, H: int, W: int, c: int) -> dict:
    """esacb200_gating_workspace_bytes's layout, restated: the experts' int header for B images (no expert axis), then B
    blocks of image_floats floats; per block the float offsets of conv3's NHWC output a3 (/4, 32 channels), the /8 maps
    x and y (64c channels) and the pool's partial sums (one row of 64c per chunk of POOL_CELLS cells), the sides h, w,
    the chunk count and the total bytes."""
    h, w = [H], [W]
    for _ in range(3):
        h.append((h[-1] + 1) // 2)
        w.append((w[-1] + 1) // 2)
    p2, p3 = h[2] * w[2], h[3] * w[3]
    chunks = -(-p3 // POOL_CELLS)
    x = _round(32 * p2)
    y = x + _round(64 * c * p3)
    part = y + _round(64 * c * p3)
    image = part + _round(64 * c * chunks)
    hdr = _round(16 + 2 * B) * 4
    return dict(h=h, w=w, chunks=chunks, hdr_bytes=hdr, a3=0, x=x, y=y, part=part, image_floats=image,
                total_bytes=hdr + B * image * 4)


def pool_partials(y: np.ndarray, capacity: int, cells=None) -> np.ndarray:
    """The pool's partial sums in float64: [chunks, 64c] from the /8 map y [P, 64c] (NHWC cells in row order), tanh first
    at capacity 1.  cells: the chunk boundaries (default: every POOL_CELLS cells)."""
    t = np.tanh(np.asarray(y, np.float64)) if capacity == 1 else np.asarray(y, np.float64)
    P = t.shape[0]
    edges = list(range(0, P, POOL_CELLS)) + [P] if cells is None else list(cells)
    return np.stack([t[a:b].sum(0) for a, b in zip(edges[:-1], edges[1:])])


def pool_bound(y: np.ndarray, capacity: int) -> np.ndarray:
    """Worst-case error of the fp32 partial sums: a chunk of n cells is a sum of n terms in some order (gamma_n, see
    expert_oracle.accumulation_bound) of values that tanhf gives to within 2 ulp, so
    2 (n + 4) 2^-24 sum|t| per channel, with n = POOL_CELLS."""
    a = np.abs(np.tanh(np.asarray(y, np.float64)) if capacity == 1 else np.asarray(y, np.float64))
    return 2 * (POOL_CELLS + 4) * 2.0 ** -24 * pool_partials(a, 2)


def head(part: np.ndarray, cells: int, sd) -> tuple:
    """The head in float64 from the partial sums part [chunks, 64c]: (log-probabilities [E], the logits z [E])."""
    p = {k: np.asarray(v, np.float64) for k, v in sd.items()}
    v = part.sum(0) / cells
    v = np.maximum(p["fc1.weight"][:, :, 0, 0] @ v + p["fc1.bias"], 0)
    v = np.maximum(p["fc2.weight"][:, :, 0, 0] @ v + p["fc2.bias"], 0)
    z = p["fc3.weight"][:, :, 0, 0] @ v + p["fc3.bias"]
    m = z.max()
    return z - m - np.log(np.exp(z - m).sum()), z


def head_bound(part: np.ndarray, cells: int, sd) -> tuple:
    """Worst-case error of the head's fp32 log-probabilities and probabilities, elementwise, from exact partial sums.
    The mean is a sum of `chunks` terms and a division (gamma_{chunks+1}); fc1 .. fc3 are FMA chains, each bounded as in
    expert_oracle.accumulation_bound (unit 2^-24) plus |W| times the input's bound.  log_softmax: the logits' errors dz
    move z_e - lse(z) by at most dz_e + max dz (lse is 1-Lipschitz in the max norm); the kernel's own roundings are z - m
    (2^-24 |z - m|), expf (2 ulp), the sum of E terms (gamma_E), logf (1 ulp of lse) and the final subtraction, all
    counted twice.  The probabilities are expf(log p): p (expm1(d) + 2^-22), d the log bound."""
    u = 2.0 ** -24
    p = {k: np.asarray(v, np.float64) for k, v in sd.items()}
    n = part.shape[0]
    v = part.sum(0) / cells
    e = 2 * (n + 2) * u * np.abs(part).sum(0) / cells
    for name in ("fc1", "fc2", "fc3"):
        Wt, b = p[name + ".weight"][:, :, 0, 0], p[name + ".bias"]
        K = Wt.shape[1]
        z = Wt @ v + b
        e = np.abs(Wt) @ e + 2 * (K + 2) * u * (np.abs(Wt) @ (np.abs(v) + e) + np.abs(b))
        v = np.maximum(z, 0) if name != "fc3" else z
    E = v.shape[0]
    m = v.max()
    lse = np.log(np.exp(v - m).sum())
    lp = v - m - lse
    own = 2 * (u * np.abs(v - m) + 2 * (E + 2) * 2 * u + u * abs(lse) + u * np.abs(v - m).max() + u * np.abs(lp))
    d = e + e.max() + own
    return d, np.exp(lp) * (np.expm1(d) + 4 * u)
