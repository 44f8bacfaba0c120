"""Argument checks of the expert stack (esac_b200/experts.py) that need no GPU: the state dicts' keys, shapes and dtypes,
the expert count, and every rejected dtype, rank, shape and device of forward_async, all raised before any device work."""
import pytest
import torch

import esac_b200.api as api
from esac_b200.experts import ExpertStack, state_dict_shapes
from oracle.expert_oracle import kaiming_state_dict


def sd():
    return kaiming_state_dict(0)


def test_state_dict_shapes_are_experts():
    shapes = state_dict_shapes()
    assert len(shapes) == 35 and list(shapes)[-1] == "mean"
    assert shapes["conv1.weight"] == (32, 3, 3, 3) and shapes["res2_skip.weight"] == (512, 256, 1, 1)
    assert shapes["fc3.weight"] == (3, 512, 1, 1) and shapes["mean"] == (3,)


@pytest.mark.parametrize("edit, match", [
    (lambda d: d.pop("fc2.bias"), "missing \\['fc2.bias'\\]"),
    (lambda d: d.pop("mean"), "missing \\['mean'\\]"),
    (lambda d: d.__setitem__("fc4.weight", torch.zeros(3, 512, 1, 1)), "unexpected \\['fc4.weight'\\]"),
    (lambda d: d.__setitem__("mean", torch.zeros(4)), "mean must be \\[3\\]"),
    (lambda d: d.__setitem__("mean", torch.zeros(1, 3)), "mean must be \\[3\\]"),
    (lambda d: d.__setitem__("mean", torch.zeros(3, dtype=torch.int64)), "mean must be a floating-point tensor"),
    (lambda d: d.__setitem__("mean", [0.0, 0.0, 0.0]), "mean must be a floating-point tensor"),
    (lambda d: d.__setitem__("conv2.weight", torch.zeros(64, 32, 1, 1)), "conv2.weight must be \\[64, 32, 3, 3\\]"),
    (lambda d: d.__setitem__("res2_skip.bias", torch.zeros(256)), "res2_skip.bias must be \\[512\\]"),
])
def test_state_dict_rejected(edit, match):
    bad = sd()
    edit(bad)
    with pytest.raises(RuntimeError, match=match):
        ExpertStack([sd(), bad], "cuda")


def test_expert_count_and_device():
    with pytest.raises(RuntimeError, match="0 experts"):
        ExpertStack([], "cuda")
    with pytest.raises(RuntimeError, match=f"{api.MAX_EXPERTS + 1} experts"):
        ExpertStack([{}] * (api.MAX_EXPERTS + 1), "cuda")
    with pytest.raises(RuntimeError, match="CUDA device"):
        ExpertStack([sd()], "cpu")


def stub(E=2):
    """An ExpertStack whose weights were never packed: enough for the checks that precede any device work."""
    s = object.__new__(ExpertStack)
    s.E, s.device, s.packed, s.workspace, s.frozen = E, torch.device("cuda", 0), None, None, False
    return s


def good(B=1, E=2, H=16, W=24):
    return torch.zeros(B, 3, H, W), torch.zeros(B, E), torch.zeros(B, E, 3, 2, 3)


@pytest.mark.parametrize("case, match", [
    ("image_float64", "expected scalar type Float but found Double \\(image\\)"),
    ("image_rank", "expected 4 dims but tensor has 3 \\(image\\)"),
    ("image_channels", "image must be \\[B,3,H,W\\]"),
    ("image_numpy", "torch CUDA tensors only \\(image is a ndarray\\)"),
    ("image_batch", "image holds 2 images for out's batch of 3"),
    ("out_half", "expected scalar type Float but found Half \\(out\\)"),
    ("out_rank", "expected 5 dims but tensor has 4 \\(out\\)"),
    ("out_size", "out must be a contiguous \\[1, 2, 3, 2, 3\\] tensor"),
    ("out_experts", "out must be a contiguous \\[1, 2, 3, 2, 3\\] tensor"),
    ("out_noncontig", "out must be a contiguous"),
    ("hist_int", "expected scalar type Float but found Int \\(hist\\)"),
    ("hist_shape", "hist must be a contiguous \\[1, 2\\] tensor"),
    ("image_noncontig", "image must be contiguous"),
    ("cpu", "takes CUDA tensors only \\(image is on the CPU\\)"),
])
def test_forward_async_rejected(case, match):
    image, hist, out = good()
    if case == "image_float64":
        image = image.double()
    elif case == "image_rank":
        image = image[0]
    elif case == "image_channels":
        image = torch.zeros(1, 4, 16, 24)
    elif case == "image_numpy":
        image = image.numpy()
    elif case == "image_batch":
        image, out = torch.zeros(2, 3, 16, 24), torch.zeros(3, 2, 3, 2, 3)
        hist = torch.zeros(3, 2)
    elif case == "out_half":
        out = out.half()
    elif case == "out_rank":
        out = out[0]
    elif case == "out_size":
        out = torch.zeros(1, 2, 3, 2, 4)      # ceil(24 / 8) = 3 columns
    elif case == "out_experts":
        out = torch.zeros(1, 3, 3, 2, 3)
    elif case == "out_noncontig":
        out = torch.zeros(1, 2, 3, 3, 2).transpose(3, 4)
    elif case == "hist_int":
        hist = hist.int()
    elif case == "hist_shape":
        hist = torch.zeros(1, 3)
    elif case == "image_noncontig":
        image = torch.zeros(1, 3, 24, 16).transpose(2, 3)
    with pytest.raises(RuntimeError, match=match):
        stub().forward_async(image, hist, out)


def test_reserve_rejects_sizes():
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        stub().reserve(0, 16, 16)
    with pytest.raises(RuntimeError, match="outside the supported range"):
        stub(E=1024).workspace_bytes(65, 16, 16)      # B * E > 65535
    with pytest.raises(RuntimeError, match="outside the supported range"):
        stub().workspace_bytes(1, 8193, 16)


def test_workspace_and_packed_sizes(lib):
    from oracle.expert_oracle import packed_floats
    for E in (1, 7, 19):
        assert lib.esacb200_experts_packed_floats(E) == packed_floats(E)
    assert lib.esacb200_experts_packed_floats(0) == -1 and lib.esacb200_experts_packed_floats(1025) == -1
    # 480x640: 32 HW floats (conv1, shared with conv3's 128 channels at /4), 64 at /2, 256 + 3 x 512 at /8; int header
    hw = 480 * 640
    per_pair = (32 * hw + 64 * hw // 4 + (256 + 3 * 512) * hw // 64) * 4
    assert lib.esacb200_experts_workspace_bytes(2, 3, 480, 640) == 256 + 6 * per_pair


def test_frozen_workspace_does_not_grow():
    s = stub()
    s.workspace, s.frozen = torch.empty(s.workspace_bytes(1, 16, 16), dtype=torch.uint8), True
    s.reserve(1, 16, 16)                       # fits: nothing to do
    with pytest.raises(RuntimeError, match="a captured graph already uses"):
        s.reserve(1, 32, 32)
