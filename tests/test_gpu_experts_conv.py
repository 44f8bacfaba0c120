"""experts_conv_kernel alone, through esacb200_test_experts_conv: every (k, stride), Cin, Cout, tile edge of the output
map, epilogue and pair layout, held bitwise to a float64 reference where the arithmetic is exact.

* Integer lattice: inputs in [-16, 16], weights in [-2, 2], integer biases and residuals.  Every partial sum is an integer
  below 2^22, which the tensor cores add exactly in any order, so the output must be the float64 reference cast to
  float32, bit for bit.
* Rounding: activations +-(1 + j 2^-12), ties included, and sparse weights in {-1, 0, 1}.  The kernel rounds its
  activations to TF32 to nearest, ties away (cvt.rna); the output must be the reference on those operands bit for bit,
  and the references on truncated, ties-to-even and unrounded operands each differ from it somewhere.
* Pairs: several experts with different weights and a mixed histogram; every float of the pair blocks outside the active
  pairs' output regions keeps its NaN sentinel, and the header holds the count, the ascending list and the flags.
"""
import numpy as np
import pytest
import torch

import esac_b200.api as api
from oracle import expert_oracle as O

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC00BAD          # a quiet NaN that no kernel writes
HDR_FILL = -7
LATTICE_LIMIT = 2 ** 22


def run_conv(B, E, hist, packed, w_off, b_off, k, stride, cin, cout, hin, win, relu, pairs, pair_floats, in_off, out_off,
             res_off, hdr):
    ctx = api._pick_ctx(pairs.device.index)
    ctx.check(ctx.lib.esacb200_test_experts_conv(
        ctx.handle, B, E, None if hist is None else hist.data_ptr(), packed.data_ptr(), w_off, b_off, k, stride, cin,
        cout, hin, win, int(relu), pairs.data_ptr(), pair_floats, in_off, out_off, res_off, hdr.data_ptr()))


def _r4(n):
    return -(-n // 4) * 4


def layer_case(B, E, hist, k, stride, cin, cout, hin, win, relu, res_mode, make_x, make_w, make_b, make_res):
    """Runs one layer on B*E pair blocks laid out [input | residual | output | slack of 128 Cout] and returns
    (pairs before, pairs after, header after, per-pair references, layout).  res_mode: 'none', 'separate', 'aliased'."""
    hout, wout = -(-hin // stride), -(-win // stride)
    in_n, out_n = hin * win * cin, hout * wout * cout
    in_off = 0
    res_off = _r4(in_n) if res_mode == "separate" else -1
    out_off = _r4(in_n) + (_r4(out_n) if res_mode == "separate" else 0)
    if res_mode == "aliased":
        res_off = out_off
    pair_floats = _r4(out_off + out_n + 128 * cout)
    n = B * E
    w = [make_w(e, (cout, k, k, cin)) for e in range(E)]
    b = [make_b(e, cout) for e in range(E)]
    w_off = 4                                    # neither segment starts at the buffer's origin
    b_off = _r4(w_off + E * w[0].size + 8)
    packed = np.zeros(b_off + E * cout + 4, np.float32)
    for e in range(E):
        packed[w_off + e * w[e].size: w_off + (e + 1) * w[e].size] = w[e].reshape(-1)
        packed[b_off + e * cout: b_off + (e + 1) * cout] = b[e]
    blocks = np.full((n, pair_floats), SENTINEL, np.uint32).view(np.float32)
    xs, rs = [], []
    for p in range(n):
        x = make_x(p, (hin, win, cin))
        blocks[p, in_off:in_off + in_n] = x.reshape(-1)
        xs.append(x)
        r = make_res(p, (hout, wout, cout)) if res_mode != "none" else None
        if r is not None:
            blocks[p, res_off:res_off + out_n] = r.reshape(-1)
        rs.append(r)
    dev = torch.device("cuda")
    pairs = torch.from_numpy(blocks.reshape(-1).copy()).to(dev)
    hdr = torch.full((16 + 2 * n,), HDR_FILL, dtype=torch.int32, device=dev)
    h = None if hist is None else torch.as_tensor(hist, dtype=torch.float32).to(dev).contiguous()
    run_conv(B, E, h, torch.from_numpy(packed).to(dev), w_off, b_off, k, stride, cin, cout, hin, win, relu, pairs,
             pair_floats, in_off, out_off, res_off, hdr)
    torch.cuda.synchronize()
    active = np.ones(n, bool) if hist is None else (np.asarray(hist, np.float32).reshape(-1) > 0)
    refs = {}
    for p in np.flatnonzero(active):
        e = p % E
        xt = torch.from_numpy(O.tf32(xs[p]).astype(np.float64)).to(dev)
        rt = None if rs[p] is None else torch.from_numpy(rs[p].astype(np.float64)).to(dev)
        refs[p] = O.conv_nhwc(xt, torch.from_numpy(w[e].astype(np.float64)).to(dev), torch.from_numpy(b[e].astype(np.float64)).to(dev),
                              stride, relu=relu, res=rt).cpu().numpy()
    return dict(before=blocks, after=pairs.cpu().numpy().reshape(n, pair_floats), hdr=hdr.cpu().numpy(), refs=refs,
                active=active, out_off=out_off, out_n=out_n, xs=xs, w=w, b=b, rs=rs, n=n)


def check_blocks(c):
    """The active pairs' output regions are their references bitwise; every other float is as it was."""
    want = c["before"].copy()
    for p, ref in c["refs"].items():
        want[p, c["out_off"]:c["out_off"] + c["out_n"]] = ref.astype(np.float32).reshape(-1)
    bad = c["after"].view(np.uint32) != want.view(np.uint32)
    if bad.any():
        p, i = np.argwhere(bad)[0]
        where = "output" if c["out_off"] <= i < c["out_off"] + c["out_n"] else "outside the output"
        raise AssertionError(f"{int(bad.sum())} floats differ; first: pair {p}, float {i} ({where}): got "
                             f"{c['after'][p, i]!r}, want {want[p, i]!r}")


def check_header(c):
    hdr, active, n = c["hdr"], c["active"], c["n"]
    on = np.flatnonzero(active)
    assert hdr[0] == len(on)
    assert (hdr[1:16] == HDR_FILL).all()
    assert np.array_equal(hdr[16:16 + len(on)], on)
    assert (hdr[16 + len(on):16 + n] == HDR_FILL).all()
    assert np.array_equal(hdr[16 + n:16 + 2 * n], active.astype(np.int32))


def lattice_makers(seed):
    rng = np.random.default_rng(seed)
    mx = lambda p, shape: rng.integers(-16, 17, shape).astype(np.float32)
    mw = lambda e, shape: rng.integers(-2, 3, shape).astype(np.float32)
    mb = lambda e, n: rng.integers(-8, 9, n).astype(np.float32)
    mr = lambda p, shape: rng.integers(-64, 65, shape).astype(np.float32)
    return mx, mw, mb, mr


def assert_lattice_premise(c):
    """Sum |w| max|x| + |b| + |res| < 2^22 for every output: partial sums are exact integers in fp32."""
    for p in c["refs"]:
        e = p % len(c["w"])
        worst = np.abs(c["w"][e]).reshape(c["w"][e].shape[0], -1).sum(1) * 16 + np.abs(c["b"][e])
        if c["rs"][p] is not None:
            worst = worst + np.abs(c["rs"][p]).max()
        assert worst.max() < LATTICE_LIMIT, worst.max()


# (k, stride, Cin, Cout, hin, win): the production layers of both networks at their shapes, and every tile edge of the
# output map (Mtot 1, 2, 127, 128, 129, 255, 256, 257, 4800), 1 x n and n x 1 maps, odd sides at stride 2, Cout 8 and 192.
CASES = [
    (3, 2, 32, 64, 31, 33),      # experts conv2, odd sides: 16 x 17
    (3, 2, 64, 128, 17, 9),      # experts conv3: 9 x 5
    (3, 2, 128, 256, 120, 160),  # experts conv4 at 480 x 640: Mtot 4800
    (3, 1, 256, 256, 60, 80),    # res1_conv1 / res1_conv3 at 480 x 640
    (1, 1, 256, 256, 1, 1),      # res1_conv2: Mtot 1
    (3, 1, 256, 512, 16, 16),    # res2_conv1: Mtot 256
    (1, 1, 512, 512, 1, 2),      # res2_conv2, res3_*, fc1, fc2: Mtot 2
    (3, 1, 512, 512, 257, 1),    # res2_conv3: Mtot 257, n x 1
    (1, 1, 256, 512, 127, 1),    # res2_skip: Mtot 127
    (1, 1, 512, 512, 8, 16),     # Mtot 128
    (3, 1, 512, 512, 3, 43),     # Mtot 129
    (3, 1, 512, 512, 15, 17),    # Mtot 255
    (3, 2, 32, 64, 15, 15),      # gating conv4, capacity 1
    (3, 2, 32, 128, 1, 513),     # gating conv4, capacity 2: 1 x 257
    (3, 1, 64, 64, 16, 8),       # gating res1_conv1 / res1_conv3, capacity 1: Mtot 128
    (1, 1, 64, 64, 129, 1),      # gating res1_conv2, capacity 1
    (3, 1, 128, 128, 1, 257),    # gating res1_conv1 / res1_conv3, capacity 2: 1 x n
    (1, 1, 128, 128, 2, 1),      # gating res1_conv2, capacity 2
    (3, 1, 64, 8, 16, 16),       # Cout 8: one warp column of one N tile
    (1, 1, 32, 192, 255, 1),     # Cout 192: a second N tile with an idle warp column
    (3, 2, 32, 192, 33, 31),     # Cout 192 at stride 2, odd sides
]
RES_MODES = ("none", "separate", "aliased")


@pytest.mark.parametrize("i", range(len(CASES)))
def test_lattice_bitwise(i):
    k, stride, cin, cout, hin, win = CASES[i]
    relu = i % 2 == 0
    res_mode = RES_MODES[i % 3]
    hist = np.array([[1.0, 0.0, 2.0], [0.0, 3.0, 1.0]], np.float32)   # pairs 0, 2, 4, 5 active: every expert
    c = layer_case(2, 3, hist, k, stride, cin, cout, hin, win, relu, res_mode, *lattice_makers(i))
    assert_lattice_premise(c)
    check_blocks(c)
    check_header(c)


@pytest.mark.parametrize("res_mode", RES_MODES)
@pytest.mark.parametrize("relu", [False, True])
def test_lattice_epilogues(relu, res_mode):
    """Every epilogue on one map with a partial last tile in both directions (Mtot 200, Cout 192)."""
    c = layer_case(1, 2, None, 3, 1, 64, 192, 10, 20, relu, res_mode, *lattice_makers(100 + relu))
    assert_lattice_premise(c)
    check_blocks(c)


def rounding_makers(seed, density):
    """Activations +-(1 + j 2^-12) with j uniform over [0, 4096) and every fourth one an exact TF32 tie (j = 2 mod 4);
    sparse weights in {-1, 0, 1}; biases and residuals on the 2^-10 grid."""
    rng = np.random.default_rng(seed)

    def mx(p, shape):
        j = rng.integers(0, 4096, shape)
        tie = rng.random(shape) < 0.25
        j = np.where(tie, (j & ~3) | 2, j)
        return (rng.choice([-1.0, 1.0], shape) * (1.0 + j * 2.0 ** -12)).astype(np.float32)
    mw = lambda e, shape: (rng.choice([-1.0, 1.0], shape) * (rng.random(shape) < density)).astype(np.float32)
    mb = lambda e, n: (rng.integers(-512, 513, n) * 2.0 ** -10).astype(np.float32)
    mr = lambda p, shape: (rng.integers(-4096, 4097, shape) * 2.0 ** -10).astype(np.float32)
    return mx, mw, mb, mr


ROUNDING_CASES = [(3, 1, 256, 64, 9, 11, "none"), (3, 2, 64, 128, 17, 16, "separate"), (1, 1, 512, 192, 5, 7, "aliased"),
                  (3, 1, 512, 8, 4, 4, "none")]


@pytest.mark.parametrize("i", range(len(ROUNDING_CASES)))
def test_activation_rounding_is_rna(i):
    k, stride, cin, cout, hin, win, res_mode = ROUNDING_CASES[i]
    c = layer_case(1, 2, None, k, stride, cin, cout, hin, win, False, res_mode, *rounding_makers(7 + i, 0.3))
    for w in c["w"]:
        assert np.abs(w).reshape(cout, -1).sum(1).max() < 2 ** 11   # sums on the 2^-10 grid stay below 2^22 units
    check_blocks(c)
    # the case tells the roundings apart: each other reference differs from rna's on some output
    for name, rnd in O.ROUNDINGS.items():
        if name == "rna":
            continue
        differs = 0
        for p, ref in c["refs"].items():
            e = p % 2
            alt = O.conv_nhwc(rnd(c["xs"][p]).astype(np.float64), c["w"][e].astype(np.float64),
                              c["b"][e].astype(np.float64), stride, relu=False,
                              res=None if c["rs"][p] is None else c["rs"][p].astype(np.float64))
            differs += O.lattice_mismatches(alt.astype(np.float32), ref)
        assert differs > 0, name


@pytest.mark.parametrize("B, E", [(1, 1), (3, 341), (4, 256), (25, 41), (1000, 3)])
def test_active_list_and_pair_blocks(B, E):
    """B*E of 1, 1023, 1024, 1025 and 3000 pairs on 1 x 1 maps: experts_active_kernel's chunk loop carries its base
    across 1024-pair chunks; every pair reads its own expert's weights and writes only its own output."""
    rng = np.random.default_rng(B * E)
    hist = (rng.random((B, E)) < 0.5) * rng.integers(1, 9, (B, E)).astype(np.float32)
    if B * E > 1:
        hist.reshape(-1)[[0, -1]] = [0.0, 4.0]
    hist[:, 0] = np.where(hist[:, 0] > 0, hist[:, 0], -1.0)       # negative counts are inactive too
    c = layer_case(B, E, hist.astype(np.float32), 1, 1, 32, 8, 1, 1, True, "separate", *lattice_makers(B + E))
    check_blocks(c)
    check_header(c)


def test_every_pair_without_histogram():
    c = layer_case(3, 4, None, 3, 2, 32, 64, 5, 3, False, "none", *lattice_makers(3))
    assert c["active"].all()
    check_blocks(c)
    check_header(c)


def test_tf32_matmul_control():
    """The exactness premise of the lattice tests, on this device through cuBLAS: integer operands of the lattice's
    ranges, K = 4608 (the widest reduction of the stack), multiplied in TF32 with fp32 accumulation, give the exact
    product.  If this fails, the bitwise lattice tests' premise is wrong, not the kernel."""
    g = torch.Generator().manual_seed(5)
    a = torch.randint(-16, 17, (4800, 4608), generator=g).float()
    b = torch.randint(-2, 3, (4608, 512), generator=g).float()
    want = (a.double() @ b.double())
    assert want.abs().max() < LATTICE_LIMIT
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        got = a.cuda() @ b.cuda()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert torch.equal(got.double().cpu(), want)


def test_refuses_outside_contract():
    dev = torch.device("cuda")
    packed = torch.zeros(4096, device=dev)
    pairs = torch.zeros(4096, device=dev)
    hdr = torch.zeros(32, dtype=torch.int32, device=dev)
    good = dict(k=3, stride=1, cin=32, cout=8, hin=2, win=2, in_off=0, out_off=128, res_off=-1, pair_floats=256,
                w_off=0, b_off=2304)

    def call(**kw):
        a = dict(good, **kw)
        ctx = api._pick_ctx(0)
        return ctx.lib.esacb200_test_experts_conv(
            ctx.handle, 1, 1, None, a.get("packed_ptr", packed.data_ptr()), a["w_off"], a["b_off"], a["k"], a["stride"],
            a["cin"], a["cout"], a["hin"], a["win"], 1, a.get("pairs_ptr", pairs.data_ptr()), a["pair_floats"],
            a["in_off"], a["out_off"], a["res_off"], hdr.data_ptr())
    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(k=2), dict(stride=3), dict(k=1, stride=2), dict(cin=48), dict(cin=0), dict(cout=7), dict(cout=0),
                dict(in_off=2), dict(out_off=130), dict(res_off=6), dict(res_off=-2), dict(pair_floats=258),
                dict(w_off=2), dict(b_off=2306), dict(out_off=240), dict(hin=0),
                dict(pairs_ptr=pairs.data_ptr() + 4), dict(packed_ptr=packed.data_ptr() + 8)):
        assert call(**bad) != 0, bad
