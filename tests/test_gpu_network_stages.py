"""Every stage of ExpertStack's and GatingNet's launch sequences, read back from their workspaces (the layouts restated in
oracle/expert_oracle.py and oracle/gating_oracle.py) after a real forward, against float64.

* Lattices, bitwise: integer images and weights in {-1, 0, 1} make the experts' conv1 and conv2 and the gating's fp32
  front end (conv1 .. conv3) exact, so a1 and a3 must be the float64 reference cast to float32 at every side in S x S.
* Seeded Kaiming networks, elementwise: each stage starts from the device's own input in the workspace, and its output
  must lie within oracle/expert_oracle.py's accumulation_bound of a float64 reference on the operands the kernel reads.
  The bound is worst-case, so it cannot fail on a correct kernel; it is there for wiring -- offsets, residual targets,
  the skip, the pool's chunks.  A stage of several layers overwrites its intermediates, and a worst-case bound carried
  through several TF32 layers grows past the values themselves, so those stages are replayed layer by layer through
  esacb200_test_experts_conv on a copy of the workspace: each layer is held to the bound on its own input, and the
  replay's last output must equal the forward's bitwise (the kernel's output does not depend on the launch around it).
"""
import functools

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.experts import LAYERS, ExpertStack
from esac_b200.gating_net import GatingNet, layers as gating_layers
from oracle import expert_oracle as O
from oracle import gating_oracle as G

pytestmark = pytest.mark.gpu

S = (1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 33, 63, 65)
SIDES = [(1, 1), (7, 9), (17, 33), (64, 80), (480, 853), (8, 1016), (8, 1024), (8, 1032)]
TC, FMA = 2.0 ** -23, 2.0 ** -24


def lattice_sd(shapes: dict, names, seed: int, base: dict) -> dict:
    """base with the layers `names` replaced by weights in {-1, 0, 1} and biases in {-1, 0, 1}."""
    g = torch.Generator().manual_seed(seed)
    sd = dict(base)
    for n in names:
        sd[n + ".weight"] = torch.randint(-1, 2, shapes[n + ".weight"], generator=g).float()
        sd[n + ".bias"] = torch.randint(-1, 2, shapes[n + ".bias"], generator=g).float()
    return sd


def lattice_image(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-2, 3, (B, 3, H, W), generator=g).float()


def smooth_image(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((B, 3, H, W), generator=g) * 1.5).contiguous()


def region(blocks, off, h, w, c):
    """[pairs, h, w, c] NHWC maps at float offset off of every block."""
    return blocks[:, off:off + h * w * c].reshape(-1, h, w, c)


def packed_w(sd, name):
    """torch [Cout, Cin, k, k] -> the kernels' [Cout, k, k, Cin], float64 on the device."""
    return torch.as_tensor(np.asarray(sd[name + ".weight"])).permute(0, 2, 3, 1).double().cuda()


def bias(sd, name):
    return torch.as_tensor(np.asarray(sd[name + ".bias"])).double().cuda()


def assert_within(got, ref, bnd, what):
    n = O.bound_violations(got, ref, bnd)
    if n:
        d = (got.double() - ref).abs()
        i = int(torch.argmax(d - bnd))
        raise AssertionError(f"{what}: {n} of {got.numel()} outside the bound; worst got "
                             f"{got.reshape(-1)[i].item()!r}, want {ref.reshape(-1)[i].item()!r} +- {bnd.reshape(-1)[i].item():.3e}")


def run_hook(B, E, packed, w_off, b_off, k, stride, cin, cout, hin, win, relu, pairs, pair_floats, in_off, out_off, res_off):
    hdr = torch.empty(16 + 2 * B * E, dtype=torch.int32, device="cuda")
    ctx = api._pick_ctx(pairs.device.index)
    ctx.check(ctx.lib.esacb200_test_experts_conv(ctx.handle, B, E, None, packed.data_ptr(), w_off, b_off, k, stride, cin, cout,
                                                 hin, win, int(relu), pairs.data_ptr(), pair_floats, in_off, out_off, res_off,
                                                 hdr.data_ptr()))


# ---------------------------------------------------------------------------------------------------------------------
# experts
# ---------------------------------------------------------------------------------------------------------------------
EXPERT_INDEX = {name: i for i, (name, *_rest) in enumerate(LAYERS)}


def expert_segments(E):
    segs, _ = O._segments(E)
    return {name: (w, b) for name, w, b, _ in segs}


def expert_blocks(st, B, H, W):
    L = O.workspace_layout(B, st.E, H, W)
    n = B * st.E * L["pair_floats"]
    return L, st.workspace[L["hdr_bytes"]:L["hdr_bytes"] + 4 * n].view(torch.float32).view(B * st.E, L["pair_floats"])


def expert_level(name):
    i = EXPERT_INDEX[name]
    return (i - 1, i) if i <= 3 else (3, 3)


@functools.lru_cache(maxsize=None)
def lattice_stack():
    from esac_b200.experts import state_dict_shapes
    shapes = state_dict_shapes()
    return ExpertStack([lattice_sd(shapes, ("conv1", "conv2"), 40 + e, O.kaiming_state_dict(50 + e)) for e in range(2)],
                       "cuda")


@pytest.mark.parametrize("H", S)
def test_experts_conv1_conv2_lattice_bitwise(H):
    st = lattice_stack()
    sds = O.unpack(st.packed.cpu().numpy(), st.E)
    for W in S:
        img = lattice_image(1, H, W, H * 100 + W)
        st.forward(img.cuda())
        torch.cuda.synchronize()
        L, blocks = expert_blocks(st, 1, H, W)
        a1 = region(blocks, L["a1"], L["h"][1], L["w"][1], 64).cpu().numpy()
        x = img.permute(0, 2, 3, 1).double().numpy()[0]
        for e, sd in enumerate(sds):
            w = lambda n: sd[n + ".weight"].transpose(0, 2, 3, 1).astype(np.float64)
            ref = O.conv_nhwc(O.conv_nhwc(x, w("conv1"), sd["conv1.bias"], 1), w("conv2"), sd["conv2.bias"], 2)
            assert np.abs(ref).max() < 2 ** 11 * 288 < 2 ** 22
            assert O.lattice_mismatches(a1[e], ref) == 0, (H, W, e)


# the launch sequence of Expert.forward after conv3: (layer, input, output, residual, ReLU)
R_STEPS = [("conv4", "a2", "r", None, True), ("res1_conv1", "r", "x", None, True), ("res1_conv2", "x", "y", None, True),
           ("res1_conv3", "y", "r", "r", True)]
S_STEPS = [("res2_conv1", "r", "x", None, True), ("res2_conv2", "x", "y", None, True), ("res2_skip", "r", "s", None, False),
           ("res2_conv3", "y", "s", "s", True), ("res3_conv1", "s", "x", None, True), ("res3_conv2", "x", "y", None, True),
           ("res3_conv3", "y", "s", "s", True)]


def check_expert_layer(blocks_in, L, sds, step, out_blocks, what):
    """out_blocks' output of `step` within the bound of the float64 layer on blocks_in's input and residual, every expert."""
    name, src, dst, res, relu = step
    _, cin, cout, k, stride = LAYERS[EXPERT_INDEX[name]]
    li, lo = expert_level(name)
    x = region(blocks_in, L[src], L["h"][li], L["w"][li], cin)
    r = None if res is None else region(blocks_in, L[res], L["h"][lo], L["w"][lo], cout)
    got = region(out_blocks, L[dst], L["h"][lo], L["w"][lo], cout)
    E = len(sds)
    for p in range(x.shape[0]):
        sd = sds[p % E]
        ref, bnd = O.bounded_layer(x[p], packed_w(sd, name), bias(sd, name), stride, relu, None if r is None else r[p],
                                   unit=TC)
        assert_within(got[p], ref, bnd, f"{what} {name} pair {p}")


def replay_experts(st, L, blocks, steps, sds, what):
    """steps through the hook on a copy of blocks, each layer held to its bound; returns the copy."""
    segs = expert_segments(st.E)
    work = blocks.clone()
    for step in steps:
        name, src, dst, res, relu = step
        _, cin, cout, k, stride = LAYERS[EXPERT_INDEX[name]]
        li, _ = expert_level(name)
        before = work.clone()
        w_off, b_off = segs[name]
        run_hook(1, st.E, st.packed, w_off, b_off, k, stride, cin, cout, L["h"][li], L["w"][li], relu, work,
                 L["pair_floats"], L[src], L[dst], -1 if res is None else L[res])
        torch.cuda.synchronize()
        check_expert_layer(before, L, sds, step, work, what)
    return work


@functools.lru_cache(maxsize=None)
def kaiming_stack(E):
    return ExpertStack([O.kaiming_state_dict(300 + e, mean=(0.5 * e, -1.0, 2.0 + e)) for e in range(E)], "cuda")


@pytest.mark.parametrize("hw", SIDES)
def test_expert_stages_within_bound(hw):
    H, W = hw
    E = 1 if H * W > 100000 else 2
    st = kaiming_stack(E)
    sds = O.unpack(st.packed.cpu().numpy(), E)
    out = st.forward(smooth_image(1, H, W, H + W).cuda())
    torch.cuda.synchronize()
    L, blocks = expert_blocks(st, 1, H, W)
    what = f"{H}x{W}"
    # a2 from a1: conv3 alone
    check_expert_layer(blocks, L, sds, ("conv3", "a1", "a2", None, True), blocks, what)
    # r from a2 and s from r: several layers, replayed
    for steps, dst in ((R_STEPS, "r"), (S_STEPS, "s")):
        work = replay_experts(st, L, blocks, steps, sds, what)
        c = 256 if dst == "r" else 512
        a, b = region(work, L[dst], L["h"][3], L["w"][3], c), region(blocks, L[dst], L["h"][3], L["w"][3], c)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (what, dst)
    # x from s (fc1), y from x (fc2)
    check_expert_layer(blocks, L, sds, ("fc1", "s", "x", None, True), blocks, what)
    check_expert_layer(blocks, L, sds, ("fc2", "x", "y", None, True), blocks, what)
    # out from y: fc3 and the mean, fp32 FMAs on unrounded operands
    y = region(blocks, L["y"], L["h"][3], L["w"][3], 512)
    for e, sd in enumerate(sds):
        mean = torch.as_tensor(sd["mean"]).double().cuda().expand(L["h"][3], L["w"][3], 3)
        ref, bnd = O.bounded_layer(y[e], packed_w(sd, "fc3"), bias(sd, "fc3"), 1, relu=False, res=mean, unit=FMA,
                                   rounding=O.tf32_none)
        assert_within(out[0, e].permute(1, 2, 0), ref, bnd, f"{what} fc3 expert {e}")


# ---------------------------------------------------------------------------------------------------------------------
# gating
# ---------------------------------------------------------------------------------------------------------------------
def gating_blocks(g, B, H, W):
    L = G.workspace_layout(B, H, W, g.capacity)
    n = B * L["image_floats"]
    return L, g.workspace[L["hdr_bytes"]:L["hdr_bytes"] + 4 * n].view(torch.float32).view(B, L["image_floats"])


@functools.lru_cache(maxsize=None)
def lattice_gating(c):
    from esac_b200.gating_net import state_dict_shapes
    E = 3
    return GatingNet(lattice_sd(state_dict_shapes(E, c), ("conv1", "conv2", "conv3"), 60 + c,
                                G.kaiming_state_dict(70 + c, E, c)), "cuda")


@pytest.mark.parametrize("c", [1, 2])
@pytest.mark.parametrize("H", S)
def test_gating_front_lattice_bitwise(H, c):
    g = lattice_gating(c)
    sd = G.unpack(g.packed.cpu().numpy(), g.E, c)
    for W in S:
        img = lattice_image(2, H, W, H * 1000 + W + c)
        g.forward(img.cuda())
        torch.cuda.synchronize()
        L, blocks = gating_blocks(g, 2, H, W)
        a3 = region(blocks, L["a3"], L["h"][2], L["w"][2], 32).cpu().numpy()
        x = img.permute(0, 2, 3, 1).double().numpy()
        for n, stride in (("conv1", 1), ("conv2", 2), ("conv3", 2)):
            x = O.conv_nhwc(x, sd[n + ".weight"].transpose(0, 2, 3, 1), sd[n + ".bias"], stride)
        assert np.abs(x).max() < 2 ** 22
        assert O.lattice_mismatches(a3, x) == 0, (H, W, c)


X_STEPS = [("conv4", "a3", "x"), ("res1_conv1", "x", "y"), ("res1_conv2", "y", "x")]


def gating_layer_check(L, sd, E, c, name, x, got, what):
    idx = [n for n, *_ in gating_layers(E, c)].index(name)
    _, cin, cout, k, stride = gating_layers(E, c)[idx]
    ref, bnd = O.bounded_layer(x, packed_w(sd, name), bias(sd, name), stride, True, unit=TC)
    assert_within(got, ref, bnd, f"{what} {name}")


def check_gating(g, img, what):
    """Every stage of one forward of g on img, from the device's own inputs."""
    B, _, H, W = img.shape
    E, c = g.E, g.capacity
    C = 64 * c
    log_p = torch.empty(B, E, device="cuda")
    prob = torch.empty(B, E, device="cuda")
    g.forward_async(img.cuda(), log_p, prob)
    torch.cuda.synchronize()
    L, blocks = gating_blocks(g, B, H, W)
    hdr = g.workspace[:L["hdr_bytes"]].view(torch.int32).cpu().numpy()
    assert hdr[0] == B and np.array_equal(hdr[16:16 + B], np.arange(B)) and (hdr[16 + B:16 + 2 * B] == 1).all(), what
    sd = G.unpack(g.packed.cpu().numpy(), E, c)
    h3, w3 = L["h"][3], L["w"][3]
    # x from a3: conv4, res1_conv1, res1_conv2, replayed through the hook with every image as a pair
    segs = {name: (w, b) for name, w, b, _ in G._segments(E, c)[0]}
    work = blocks.clone()
    for name, src, dst in X_STEPS:
        _, cin, cout, k, stride = next(l for l in gating_layers(E, c) if l[0] == name)
        lvl = 2 if name == "conv4" else 3
        x = region(work, L[src], L["h"][lvl], L["w"][lvl], cin).clone()
        run_hook(B, 1, g.packed, segs[name][0], segs[name][1], k, stride, cin, cout, L["h"][lvl], L["w"][lvl], True, work,
                 L["image_floats"], L[src], L[dst], -1)
        torch.cuda.synchronize()
        gating_layer_check(L, sd, E, c, name, x, region(work, L[dst], h3, w3, cout), what)
    a, b = region(work, L["x"], h3, w3, C), region(blocks, L["x"], h3, w3, C)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what
    # y from x: res1_conv3
    y = region(blocks, L["y"], h3, w3, C)
    gating_layer_check(L, sd, E, c, "res1_conv3", region(blocks, L["x"], h3, w3, C), y, what)
    # the pool's partial sums from y, and the head from the partial sums
    part = blocks[:, L["part"]:L["part"] + L["chunks"] * C].reshape(B, L["chunks"], C).cpu().numpy()
    yn = y.reshape(B, h3 * w3, C).cpu().numpy()
    lp, pr = log_p.cpu().numpy(), prob.cpu().numpy()
    for i in range(B):
        ref, bnd = G.pool_partials(yn[i], c), G.pool_bound(yn[i], c)
        assert O.bound_violations(part[i], ref, bnd) == 0, (what, "pool", i)
        ref_lp, _ = G.head(part[i].astype(np.float64), h3 * w3, sd)
        d_lp, d_p = G.head_bound(part[i].astype(np.float64), h3 * w3, sd)
        assert O.bound_violations(lp[i], ref_lp, d_lp) == 0, (what, "log_softmax", i, lp[i] - ref_lp, d_lp)
        assert O.bound_violations(pr[i], np.exp(ref_lp), d_p) == 0, (what, "probabilities", i)


@functools.lru_cache(maxsize=None)
def kaiming_gating(E, c):
    return GatingNet(G.kaiming_state_dict(500 + E + c, E, c), "cuda")


@pytest.mark.parametrize("c", [1, 2])
@pytest.mark.parametrize("hw", SIDES)
def test_gating_stages_within_bound(hw, c):
    H, W = hw
    check_gating(kaiming_gating(7, c), smooth_image(2, H, W, H * W + c), f"{H}x{W} c={c}")


@pytest.mark.parametrize("E, c", [(1, 1), (255, 2), (256, 1), (257, 2), (1024, 1)])
def test_gating_head_expert_counts(E, c):
    """E above 256 runs the head's e += 256 loops; E = 1024 is the largest the head's shared logits hold."""
    check_gating(kaiming_gating(E, c), smooth_image(2, 17, 33, E), f"E={E} c={c}")


def test_gating_image_list_beyond_one_chunk():
    """1100 images: experts_active_kernel lists them in two chunks of 1024."""
    check_gating(kaiming_gating(5, 1), smooth_image(1100, 8, 8, 3), "B=1100")
