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
