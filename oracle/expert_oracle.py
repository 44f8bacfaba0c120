"""Oracle for the expert stack (esac_b200/experts.py, esac_b200/csrc/experts.cu).  TEST INFRASTRUCTURE ONLY.

`forward` is the reference's Expert (code/expert.py) written from its layer table as float64 torch.nn.functional calls on
the CPU: conv1 .. conv4 with ReLU, three residual blocks -- res + ReLU(conv) twice, and res2_skip(res) + ReLU(conv) in the
second -- fc1, fc2 with ReLU, fc3, plus the expert's mean.  `pack` / `unpack` restate the packed weight layout of
include/esac_b200.h in numpy, with the TF32 rounding (cvt.rna: to nearest, ties away from zero) of the layers the tensor
cores read.

Only tests/, tools/ and examples/ may import this module; the product path never does.
"""
from __future__ import annotations

import numpy as np

from esac_b200.experts import LAYERS, state_dict_shapes

ALIGN = 64  # floats: every segment of the packed weights starts on this boundary


def apply(x, p: dict):
    """Expert.forward on x [B,3,H,W] with parameters p (key -> tensor, on x's device and dtype), as functional calls."""
    import torch.nn.functional as F
    layer = {name: (k, s) for name, _, _, k, s in LAYERS}

    def conv(name, v):
        k, s = layer[name]
        return F.conv2d(v, p[name + ".weight"], p[name + ".bias"], stride=s, padding=k // 2)

    x = F.relu(conv("conv1", x))
    x = F.relu(conv("conv2", x))
    x = F.relu(conv("conv3", x))
    res = F.relu(conv("conv4", x))
    x = F.relu(conv("res1_conv3", F.relu(conv("res1_conv2", F.relu(conv("res1_conv1", res))))))
    res = res + x
    x = F.relu(conv("res2_conv3", F.relu(conv("res2_conv2", F.relu(conv("res2_conv1", res))))))
    res = conv("res2_skip", res) + x
    x = F.relu(conv("res3_conv3", F.relu(conv("res3_conv2", F.relu(conv("res3_conv1", res))))))
    res = res + x
    x = conv("fc3", F.relu(conv("fc2", F.relu(conv("fc1", res)))))
    return x + p["mean"].view(1, 3, 1, 1)


def forward(image, sd):
    """Expert.forward of one expert on image [B,3,H,W], in float64 on the CPU.  sd: the expert's state dict."""
    import torch
    p = {k: torch.as_tensor(v).detach().to("cpu", torch.float64) for k, v in sd.items()}
    return apply(torch.as_tensor(image).detach().to("cpu", torch.float64), p)


def tf32(a: np.ndarray) -> np.ndarray:
    """float32 values rounded to TF32 (10 mantissa bits) to nearest, ties away from zero; finite inputs."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _round(n: int) -> int:
    return -(-n // ALIGN) * ALIGN


def _segments(E: int):
    """(name, W offset, b offset, (Cout, Cin, k)) per layer, and the mean's offset."""
    off, out = 0, []
    for name, cin, cout, k, _ in LAYERS:
        w = off
        off += _round(E * cout * cin * k * k)
        out.append((name, w, off, (cout, cin, k)))
        off += _round(E * cout)
    return out, off


def packed_floats(E: int) -> int:
    return _segments(E)[1] + _round(3 * E)


def pack(sds) -> np.ndarray:
    """The packed float32 weights of the experts with state dicts `sds`."""
    E = len(sds)
    segs, mean_off = _segments(E)
    out = np.zeros(packed_floats(E), np.float32)
    for name, w_off, b_off, (cout, cin, k) in segs:
        gemm = name not in ("conv1", "fc3")
        for e, sd in enumerate(sds):
            w = np.asarray(sd[name + ".weight"].detach().cpu(), np.float32).transpose(0, 2, 3, 1).reshape(-1)
            n = w.size
            out[w_off + e * n: w_off + (e + 1) * n] = tf32(w) if gemm else w
            out[b_off + e * cout: b_off + (e + 1) * cout] = np.asarray(sd[name + ".bias"].detach().cpu(), np.float32)
    for e, sd in enumerate(sds):
        out[mean_off + 3 * e: mean_off + 3 * e + 3] = np.asarray(sd["mean"].detach().cpu(), np.float32)
    return out


def unpack(packed: np.ndarray, E: int) -> list:
    """The E state dicts (numpy float32, torch's layouts) held by packed weights."""
    segs, mean_off = _segments(E)
    sds = [{} for _ in range(E)]
    for name, w_off, b_off, (cout, cin, k) in segs:
        n = cout * cin * k * k
        for e in range(E):
            w = packed[w_off + e * n: w_off + (e + 1) * n].reshape(cout, k, k, cin).transpose(0, 3, 1, 2)
            sds[e][name + ".weight"] = np.ascontiguousarray(w)
            sds[e][name + ".bias"] = packed[b_off + e * cout: b_off + (e + 1) * cout].copy()
    for e in range(E):
        sds[e]["mean"] = packed[mean_off + 3 * e: mean_off + 3 * e + 3].copy()
    assert all(list(sd) == list(state_dict_shapes()) for sd in sds)
    return sds


def kaiming_state_dict(seed: int, mean=(0.0, 0.0, 0.0)) -> dict:
    """A seeded Kaiming-normal (fan-in, ReLU gain) expert with small uniform biases: activations keep their scale
    through the 19 layers, as in a trained network."""
    import torch
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in state_dict_shapes().items():
        if name == "mean":
            sd[name] = torch.tensor(mean, dtype=torch.float32)
        elif name.endswith(".weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            sd[name] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        else:
            sd[name] = (torch.rand(shape, generator=g) - 0.5) * 0.1
    return sd
