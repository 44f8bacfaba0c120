"""The oracles behind tests/test_gpu_experts_conv.py and tests/test_gpu_network_stages.py, on the CPU: the restated
workspace layouts against the library's own sizes, the TF32 roundings on known values, and mutants of each layer,
emulated in numpy, that the tests' comparators must reject -- unrounded or truncated activations, an off-by-one halo,
the residual added before the ReLU, another expert's weights, one wrong pool chunk."""
import numpy as np
import pytest
import torch

from oracle import expert_oracle as O
from oracle import gating_oracle as G

TC = 2.0 ** -23


def test_expert_workspace_layout_matches_library(lib):
    for B, E, H, W in [(1, 1, 1, 1), (1, 2, 7, 9), (3, 5, 17, 33), (1, 7, 480, 640), (2, 19, 480, 853), (1, 1, 8, 1032),
                       (1000, 3, 8, 8), (4, 256, 65, 63), (1, 1, 8192, 1)]:
        L = O.workspace_layout(B, E, H, W)
        assert L["total_bytes"] == lib.esacb200_experts_workspace_bytes(B, E, H, W), (B, E, H, W)
        assert L["a1"] >= max(32 * H * W, 128 * L["h"][2] * L["w"][2])
        order = [L["a1"], L["r"], L["s"], L["x"], L["y"], L["pair_floats"]]
        assert order == sorted(order) and all(o % 64 == 0 for o in order)


def test_gating_workspace_layout_matches_library(lib):
    for B, E, c, H, W in [(1, 1, 1, 1, 1), (2, 7, 1, 7, 9), (2, 50, 2, 17, 33), (1, 7, 2, 480, 853), (1100, 5, 1, 8, 8),
                          (3, 1024, 2, 8, 1016), (1, 3, 1, 8, 1024), (1, 3, 2, 8, 1032)]:
        L = G.workspace_layout(B, H, W, c)
        assert L["total_bytes"] == lib.esacb200_gating_workspace_bytes(B, E, c, H, W), (B, E, c, H, W)
        assert L["chunks"] == -(-L["h"][3] * L["w"][3] // 128)
    assert [G.workspace_layout(1, 8, n, 1)["chunks"] for n in (1016, 1024, 1032)] == [1, 1, 2]


def test_tf32_roundings_on_known_values():
    one = np.float32(1.0)
    ulp = 2.0 ** -10
    x = np.array([1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -12, 1 + 3 * 2 ** -12, -(1 + 2 ** -11)], np.float32)
    assert O.tf32(x).tolist() == [1 + ulp, 1 + 2 * ulp, 1, 1 + ulp, -(1 + ulp)]            # ties away from zero
    assert O.tf32_rne(x).tolist() == [1, 1 + 2 * ulp, 1, 1 + ulp, -1.0]                     # ties to even
    assert O.tf32_rz(x).tolist() == [1, 1 + ulp, 1, 1, -1.0]                                # toward zero
    assert np.array_equal(O.tf32_none(x), x) and O.tf32(one) == one
    t = torch.from_numpy(x)
    for name, f in O.ROUNDINGS.items():
        assert np.array_equal(O._tf32_torch(t, f).numpy(), f(x)), name


def rounding_layer(seed=0, cin=64, cout=32, hw=(6, 7), k=3):
    rng = np.random.default_rng(seed)
    j = rng.integers(0, 4096, hw + (cin,))
    j = np.where(rng.random(j.shape) < 0.25, (j & ~3) | 2, j)
    x = (rng.choice([-1.0, 1.0], j.shape) * (1 + j * 2.0 ** -12)).astype(np.float32)
    w = (rng.choice([-1.0, 1.0], (cout, k, k, cin)) * (rng.random((cout, k, k, cin)) < 0.3)).astype(np.float32)
    b = (rng.integers(-64, 65, cout) * 2.0 ** -10).astype(np.float32)
    return x, w, b


@pytest.mark.parametrize("mutant", ["none", "rz", "rne"])
def test_lattice_comparator_rejects_other_activation_roundings(mutant):
    x, w, b = rounding_layer()
    ref = O.conv_nhwc(O.tf32(x).astype(np.float64), w, b, 1, relu=False)
    assert O.lattice_mismatches(ref.astype(np.float32), ref) == 0
    bad = O.conv_nhwc(O.ROUNDINGS[mutant](x).astype(np.float64), w, b, 1, relu=False).astype(np.float32)
    assert O.lattice_mismatches(bad, ref) > 0


def kaiming_layer(seed, cin=64, cout=64, hw=(9, 11), k=3, E=2):
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.standard_normal(hw + (cin,)), 0).astype(np.float32)
    ws = [O.tf32((rng.standard_normal((cout, k, k, cin)) * (2.0 / (cin * k * k)) ** 0.5).astype(np.float32))
          for _ in range(E)]
    bs = [((rng.random(cout) - 0.5) * 0.1).astype(np.float32) for _ in range(E)]
    res = rng.standard_normal(hw[:2] + (cout,)).astype(np.float32)
    return x, ws, bs, res


def fp32_device(x, w, b, stride, relu, res):
    """A correct layer as an fp32 device computes it: TF32 operands, float32 accumulation (torch on the CPU)."""
    import torch.nn.functional as F
    xt = torch.from_numpy(O.tf32(x)).permute(2, 0, 1)[None]
    wt = torch.from_numpy(w).permute(0, 3, 1, 2)
    y = F.conv2d(xt, wt, torch.from_numpy(b), stride=stride, padding=w.shape[1] // 2)[0].permute(1, 2, 0)
    if relu:
        y = torch.relu(y)
    if res is not None:
        y = torch.from_numpy(res) + y
    return y.numpy()


@pytest.mark.parametrize("stride", [1, 2])
def test_bound_admits_a_correct_fp32_layer(stride):
    x, ws, bs, res = kaiming_layer(1)
    r = None if stride == 2 else res
    got = fp32_device(x, ws[0], bs[0], stride, True, r)
    ref, bnd = O.bounded_layer(x, ws[0].astype(np.float64), bs[0].astype(np.float64), stride, True, r, unit=TC)
    assert O.bound_violations(got, ref, bnd) == 0
    assert O.lattice_mismatches(got, ref) > 0          # not exact: the bound, not bitwise equality, is the check here


def lattice_layer(seed, cin=32, cout=16, hw=(7, 9), k=3, E=2):
    rng = np.random.default_rng(seed)
    x = rng.integers(-16, 17, hw + (cin,)).astype(np.float32)
    ws = [rng.integers(-2, 3, (cout, k, k, cin)).astype(np.float32) for _ in range(E)]
    bs = [rng.integers(-8, 9, cout).astype(np.float32) for _ in range(E)]
    res = rng.integers(-64, 65, hw[:2] + (cout,)).astype(np.float32)
    return x, ws, bs, res


def both_reject(bad, x, w, b, stride, relu, res):
    """The bitwise comparator of the lattice tests and the bound comparator of the stage tests both reject `bad`."""
    ref = O.conv_nhwc(x.astype(np.float64), w, b, stride, relu=relu, res=res)
    assert O.lattice_mismatches(ref.astype(np.float32), ref) == 0
    _, bnd = O.bounded_layer(x, w.astype(np.float64), b.astype(np.float64), stride, relu, res, unit=TC)
    assert O.lattice_mismatches(bad, ref) > 0
    assert O.bound_violations(bad, ref, bnd) > 0


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("edge", ["top", "bottom", "left", "right"])
def test_comparators_reject_an_off_by_one_halo(stride, edge):
    """The input window one pixel off along one edge: the row or column that should be zero padding is read from the
    image (or the last one is lost)."""
    for make in (lattice_layer, kaiming_layer):
        x, ws, bs, res = make(2)
        pad = {"top": ((2, 0), (1, 1)), "bottom": ((0, 2), (1, 1)), "left": ((1, 1), (2, 0)), "right": ((1, 1), (0, 2))}[edge]
        xp = np.pad(x.astype(np.float64), pad + ((0, 0),))
        w = ws[0].astype(np.float64)
        wt = torch.from_numpy(w).permute(0, 3, 1, 2)
        y = torch.nn.functional.conv2d(torch.from_numpy(xp).permute(2, 0, 1)[None], wt, torch.from_numpy(bs[0].astype(np.float64)),
                                       stride=stride)[0].permute(1, 2, 0)
        ho, wo = -(-x.shape[0] // stride), -(-x.shape[1] // stride)
        bad = torch.relu(y[:ho, :wo]).numpy().astype(np.float32)
        if make is lattice_layer:
            both_reject(bad, x, ws[0], bs[0], stride, True, None)
        else:
            ref, bnd = O.bounded_layer(x, w, bs[0].astype(np.float64), stride, True, unit=TC)
            assert O.bound_violations(bad, ref, bnd) > 0


def test_comparators_reject_the_residual_before_the_relu():
    for make in (lattice_layer, kaiming_layer):
        x, ws, bs, res = make(3)
        pre = O.conv_nhwc(O.tf32(x).astype(np.float64), ws[0], bs[0], 1, relu=False)
        bad = np.maximum(pre + res, 0).astype(np.float32)
        ref, bnd = O.bounded_layer(x, ws[0].astype(np.float64), bs[0].astype(np.float64), 1, True, res, unit=TC)
        assert O.bound_violations(bad, ref, bnd) > 0
        if make is lattice_layer:
            both_reject(bad, x, ws[0], bs[0], 1, True, res)


def test_comparators_reject_another_experts_weights():
    for make in (lattice_layer, kaiming_layer):
        x, ws, bs, res = make(4)
        bad = O.conv_nhwc(O.tf32(x).astype(np.float64), ws[1], bs[1], 2).astype(np.float32)
        ref, bnd = O.bounded_layer(x, ws[0].astype(np.float64), bs[0].astype(np.float64), 2, True, unit=TC)
        assert O.bound_violations(bad, ref, bnd) > 0
        if make is lattice_layer:
            both_reject(bad, x, ws[0], bs[0], 2, True, None)


def test_pool_and_head_comparators_reject_one_wrong_chunk():
    """One chunk boundary a cell off: the pool's comparator rejects it (the head sees only the total, which it keeps).
    One chunk's sum lost, or one chunk summed twice: both comparators reject it.  The correct partial sums in fp32 pass
    both."""
    rng = np.random.default_rng(5)
    E, c = 9, 1
    sd = {k: v.numpy() for k, v in G.kaiming_state_dict(6, E, c).items()}
    P = 300
    y = (rng.standard_normal((P, 64 * c)) * 2).astype(np.float32)
    good = G.pool_partials(y, c)
    assert good.shape[0] == 3
    bnd = G.pool_bound(y, c)
    ref_lp, _ = G.head(good, P, sd)
    d_lp, _ = G.head_bound(good, P, sd)
    ok = good.astype(np.float32)
    assert O.bound_violations(ok, good, bnd) == 0
    assert O.bound_violations(G.head(ok.astype(np.float64), P, sd)[0], ref_lp, d_lp) == 0
    shifted = G.pool_partials(y, c, cells=[0, 129, 256, P]).astype(np.float32)
    dropped = good.copy()
    dropped[1] = 0
    twice = good.copy()
    twice[2] = good[1]
    assert O.bound_violations(shifted, good, bnd) > 0
    for bad in (dropped.astype(np.float32), twice.astype(np.float32)):
        assert O.bound_violations(bad, good, bnd) > 0
        assert O.bound_violations(G.head(bad.astype(np.float64), P, sd)[0], ref_lp, d_lp) > 0
