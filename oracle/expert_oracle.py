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


def tf32_rz(a: np.ndarray) -> np.ndarray:
    """float32 values truncated to TF32 (round toward zero): what the tensor cores read from fp32 bits left unrounded."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rne(a: np.ndarray) -> np.ndarray:
    """float32 values rounded to TF32 to nearest, ties to even; finite inputs."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    odd = (u >> np.uint32(13)) & np.uint32(1)
    return ((u + np.uint32(0xFFF) + odd) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_none(a: np.ndarray) -> np.ndarray:
    """float32 values as they are: full fp32 operands."""
    return np.ascontiguousarray(a, np.float32).copy()


# The operand roundings a tensor-core layer could apply to its fp32 activations; the kernels use "rna".
ROUNDINGS = {"rna": tf32, "rz": tf32_rz, "rne": tf32_rne, "none": tf32_none}


def conv_nhwc(x, w, b, stride: int, relu: bool = True, res=None):
    """One layer of the stack in float64: res + ReLU(conv(x, w) + b), with zero padding k // 2.  x [..., H, W, Cin]
    (NHWC, leading axes are images), w [Cout, k, k, Cin] (the packed layout of one expert), b [Cout] or None, res
    [..., Hout, Wout, Cout] or None.  numpy in, numpy out; torch tensors stay on their device."""
    import torch
    import torch.nn.functional as F
    as_np = not isinstance(x, torch.Tensor)
    t = lambda v: torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v).to(torch.float64)
    xt = t(x)
    dev = xt.device
    lead = xt.shape[:-3]
    wt = t(w).to(dev).permute(0, 3, 1, 2)
    k = int(wt.shape[-1])
    xin = xt.reshape((-1,) + tuple(xt.shape[-3:])).permute(0, 3, 1, 2)
    y = F.conv2d(xin, wt, None if b is None else t(b).to(dev), stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    y = y.reshape(tuple(lead) + tuple(y.shape[1:]))
    if relu:
        y = torch.relu(y)
    if res is not None:
        y = y + t(res).to(dev)
    return y.cpu().numpy() if as_np else y


def accumulation_bound(absx, absw, absb, stride: int, unit: float, absres=None):
    """Worst-case error of one layer's fp32 output, elementwise, given exact operands x~ (what the layer multiplies: TF32
    values for the tensor cores, fp32 ones for the FMA kernels) and float64 arithmetic for the reference:

        |fl(res + ReLU(sum_k w_k x~_k + b)) - (res + ReLU(sum_k w_k x~_k + b))|
            <= 2 (K + 2) unit (sum_k |w_k| |x~_k| + |b| + |res|).

    Derivation.  A product of two TF32 values has at most 22 significant bits, so the tensor cores form it exactly; an
    FMA rounds once per step.  Summing K terms in any order (any tree, any grouping into MMA k-steps) with a relative
    error of at most `unit` per addition is off by at most gamma_K * sum|terms| (Higham, Accuracy and Stability of
    Numerical Algorithms, eq. 4.4), gamma_K = K unit / (1 - K unit) <= 2 K unit while K unit <= 1/2.  Adding the bias
    and then the residual are two more roundings, each at most `unit` times |sum| + |b| + |res|.  ReLU is 1-Lipschitz.
    `unit` is 2^-24 for round-to-nearest fp32 (the FMA kernels) and 2^-23 for the tensor cores, whose adds are allowed
    to truncate.  The bound holds for any accumulation order, so it cannot fail on a correct kernel; it is loose (a
    random-sign sum errs about sqrt(K) unit), which makes it a check of wiring -- offsets, operands, residual targets
    -- not of rounding.  absx |x~| NHWC, absw |w| [Cout, k, k, Cin], absb |b| or None, absres |res| or None."""
    K = int(np.prod(absw.shape[1:]))
    assert K * unit <= 0.5
    return 2 * (K + 2) * unit * conv_nhwc(absx, absw, absb, stride, relu=False, res=absres)


def bounded_layer(x, w, b, stride: int, relu: bool = True, res=None, unit: float = 2.0 ** -23, rounding=tf32):
    """One layer on the device's own input x (fp32 NHWC, numpy or torch): (float64 reference, elementwise bound) of its
    fp32 output.  The reference multiplies rounding(x) -- the operand the tensor cores read; pass tf32_none and
    unit 2^-24 for the FMA kernels -- by w [Cout, k, k, Cin] as packed, adds b, applies the ReLU and adds res; the bound is
    accumulation_bound's."""
    import torch
    if isinstance(x, torch.Tensor):
        xr = _tf32_torch(x, rounding).to(torch.float64)
        w, b = torch.as_tensor(w).to(x.device), None if b is None else torch.as_tensor(b).to(x.device)
        res = None if res is None else torch.as_tensor(res).to(x.device)
    else:
        xr = rounding(np.asarray(x, np.float32)).astype(np.float64)
    val = conv_nhwc(xr, w, b, stride, relu=relu, res=res)
    bnd = accumulation_bound(abs(xr), abs(w), None if b is None else abs(b), stride, unit, None if res is None else abs(res))
    return val, bnd


def _tf32_torch(x, rounding):
    """rounding (tf32, tf32_rz, tf32_rne or tf32_none) on a float32 torch tensor, on its device."""
    import torch
    u = x.to(torch.float32).contiguous().view(torch.int32)
    mask = torch.tensor(-8192, dtype=torch.int32, device=x.device)  # 0xFFFFE000
    if rounding is tf32:
        u = (u + 0x1000) & mask
    elif rounding is tf32_rz:
        u = u & mask
    elif rounding is tf32_rne:
        u = (u + 0xFFF + ((u >> 13) & 1)) & mask
    elif rounding is not tf32_none:
        raise ValueError(rounding)
    return u.view(torch.float32)


def _np(a):
    return a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)


def lattice_mismatches(got, ref64) -> int:
    """Elements of a float32 result that are not bitwise the float64 reference cast to float32."""
    want = np.asarray(_np(ref64), np.float64).astype(np.float32)
    return int(np.count_nonzero(np.asarray(_np(got), np.float32).view(np.uint32) != want.view(np.uint32)))


def bound_violations(got, ref, bound) -> int:
    """Elements farther from the reference than their bound (a NaN counts)."""
    d = np.abs(np.asarray(_np(got), np.float64) - np.asarray(_np(ref), np.float64))
    return int(np.count_nonzero(~(d <= _np(bound))))


def workspace_layout(B: int, E: int, H: int, W: int) -> dict:
    """esacb200_experts_workspace_bytes's layout, restated: the int header's bytes (active count, ascending list of b*E+e,
    B*E flags), then B*E blocks of pair_floats floats; per block the NHWC activations' float offsets (a0 and a2 share
    offset 0), the sides h, w of the four resolutions and the total bytes."""
    h, w = [H], [W]
    for _ in range(3):
        h.append((h[-1] + 1) // 2)
        w.append((w[-1] + 1) // 2)
    p = [h[i] * w[i] for i in range(4)]
    r64 = _round
    a1 = r64(max(32 * p[0], 128 * p[2]))
    r = a1 + r64(64 * p[1])
    s_ = r + r64(256 * p[3])
    x = s_ + r64(512 * p[3])
    y = x + r64(512 * p[3])
    pair = y + r64(512 * p[3])
    hdr = r64(16 + 2 * B * E) * 4
    return dict(h=h, w=w, hdr_bytes=hdr, a0=0, a1=a1, a2=0, r=r, s=s_, x=x, y=y, pair_floats=pair,
                total_bytes=hdr + B * E * pair * 4)


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
