"""The gating network on the device (esac_b200/gating_net.py, esac_b200/csrc/gating_net.cu): the packed weights, accuracy
against the float64 oracle (oracle/gating_oracle.py) next to cuDNN's TF32 route, invariance of each image's output to the
batch and the run, capture against eager, and the expert stack's outputs held to those it computed before the gating
network shared its convolution kernel."""
import functools
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from esac_b200.experts import ExpertStack
from esac_b200.gating_net import GatingNet
from oracle import expert_oracle as XO
from oracle import gating_oracle as O

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu

# Absolute floor of the accuracy check: below it, a log-probability error is fp32 rounding of the logits, not the
# route's numerics (the logits are O(1); E = 1 gives 0 exactly on both routes).
FLOOR = 2e-5


def image_like(B, H, W, seed):
    """Smooth random images in [0, 1] with noise, normalised as the room datasets do ((x - 0.4) / 0.25)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand((B, 3, max(1, H // 16), max(1, W // 16)), generator=g)
    x = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)
    x = (x + 0.05 * torch.randn((B, 3, H, W), generator=g)).clamp(0, 1)
    return ((x - 0.4) / 0.25).contiguous()


@functools.lru_cache(maxsize=None)
def weights(E, c):
    return O.kaiming_state_dict(1000 + 10 * E + c, E, c)


@functools.lru_cache(maxsize=None)
def net(E, c):
    return GatingNet(weights(E, c), "cuda")


def torch_tf32(E, c, image):
    """The reference's route on the device: the Gating module in float32 under cuDNN's TF32 default."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        m = O.make_gating_class()(E, c).cuda()
        m.load_state_dict(weights(E, c))
        with torch.no_grad():
            return m(image.cuda())
    finally:
        torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("E, c", [(7, 1), (50, 2)])
def test_pack_matches_oracle(E, c):
    got = net(E, c).packed.cpu().numpy()
    want = O.pack(weights(E, c), c)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("c", [1, 2])
@pytest.mark.parametrize("hw", [(480, 640), (480, 853), (640, 480), (64, 80)])
@pytest.mark.parametrize("E", [1, 7, 50])
def test_accuracy_against_oracle(E, c, hw):
    H, W = hw
    img = image_like(2, H, W, seed=H + W + c)
    ours = net(E, c).forward(img.cuda())
    torch.cuda.synchronize()
    assert ours.shape == (2, E)
    ref = O.forward(img, weights(E, c), c)
    e_ours = float((ours.double().cpu() - ref).abs().max())
    e_torch = float((torch_tf32(E, c, img).double().cpu() - ref).abs().max())
    print(f"E={E} c={c} {H}x{W}: GatingNet {e_ours:.3e}, cuDNN TF32 {e_torch:.3e}")
    assert torch.isfinite(ours).all()
    assert e_ours <= max(2 * e_torch, FLOOR), (E, c, H, W, e_ours, e_torch)


@pytest.mark.parametrize("E, c, hw", [(7, 1, (120, 168)), (50, 2, (96, 131))])
def test_batch_and_run_invariance(E, c, hw):
    g = net(E, c)
    imgs = image_like(8, *hw, seed=E).cuda()
    alone = [g.forward(imgs[b:b + 1].contiguous()) for b in range(8)]
    for B in (1, 3, 8):
        for first in range(0, 8, B):
            out = g.forward(imgs[first:first + B].contiguous())
            for b in range(min(B, 8 - first)):
                assert torch.equal(out[b], alone[first + b][0]), (B, first, b)
    shuffled = g.forward(imgs.flip(0).contiguous())
    assert torch.equal(shuffled.flip(0), torch.cat(alone))
    assert torch.equal(g.forward(imgs), g.forward(imgs))


def test_probabilities_are_exp_of_log_probabilities():
    g = net(19, 1)
    img = image_like(3, 64, 88, seed=4).cuda()
    log_p = torch.empty(3, 19, device="cuda")
    probs = torch.empty(3, 19, device="cuda")
    g.forward_async(img, log_p, probs)
    assert torch.equal(log_p, g.forward(img))
    assert torch.allclose(probs, log_p.exp(), rtol=2e-7, atol=0)
    assert torch.allclose(probs.sum(1).double(), torch.ones(3, dtype=torch.float64, device="cuda"), atol=1e-5)


def test_capture_replays_without_host_synchronisation():
    E, c, H, W = 10, 2, 120, 160
    g = GatingNet(weights(E, c), "cuda")        # its own: the capture freezes its workspace
    img = image_like(2, H, W, seed=8).cuda()
    log_p = torch.full((2, E), float("nan"), device="cuda")
    probs = torch.full((2, E), float("nan"), device="cuda")
    g.reserve(2, H, W)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g.forward_async(img, log_p, probs)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g.forward_async(img, log_p, probs)
    for seed in (8, 9, 10):
        img.copy_(image_like(2, H, W, seed=seed))
        log_p.fill_(float("nan"))
        graph.replay()
        want = torch.empty_like(log_p)
        want_p = torch.empty_like(probs)
        g.forward_async(img, want, want_p)
        torch.cuda.synchronize()
        assert torch.equal(log_p, want) and torch.equal(probs, want_p), seed
    stream = torch.cuda.current_stream()
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))       # ~1 s of device time ahead of the replay
    graph.replay()
    assert not stream.query(), "graph.replay() waited for the device"
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="a captured graph already uses"):
        g.forward(image_like(1, 4 * H, W, seed=1).cuda())


def test_capture_needs_reserved_workspace():
    g = GatingNet(weights(7, 1), "cuda")
    img = image_like(1, 64, 64, seed=1).cuda()
    out = torch.empty((1, 7), device="cuda")
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="reserve"):
        with torch.cuda.graph(graph):
            g.forward_async(img, out)


def test_expert_stack_outputs_unchanged():
    """ExpertStack's predictions on seeded inputs, bitwise those written by the expert stack before its convolution kernel
    took the gating network's layers (tests/golden/experts/stack_parent.npz)."""
    golden = np.load(ROOT / "tests" / "golden" / "experts" / "stack_parent.npz")
    E = 3
    st = ExpertStack([XO.kaiming_state_dict(100 + e, mean=(0.5 * e, -1.0, 2.0 + e)) for e in range(E)], "cuda")
    a = st.forward(image_like(2, 64, 80, seed=11).cuda(), torch.tensor([[1.0, 0.0, 2.0], [0.0, 5.0, 1.0]], device="cuda"))
    b = st.forward(image_like(1, 120, 168, seed=12).cuda())
    assert np.array_equal(a.cpu().numpy().view(np.uint32), golden["a"].view(np.uint32))
    assert np.array_equal(b.cpu().numpy().view(np.uint32), golden["b"].view(np.uint32))
