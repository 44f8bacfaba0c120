"""The expert stack on the device (esac_b200/experts.py, esac_b200/csrc/experts.cu): accuracy against the float64 oracle
(oracle/expert_oracle.py) next to cuDNN's TF32 route, invariance of each pair's output to the active set, the batch and
graph replays, zero planes for inactive experts, capture against eager, and the captured test step of
examples/test_step_expert_stack_graph_synthetic.py."""
import functools
import importlib.util
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from esac_b200.experts import ExpertStack, prediction_size
from oracle import expert_oracle as O

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


def image_like(B, H, W, seed):
    """Smooth random images in [0, 1] with noise, normalised as the datasets do ((x - 0.4) / 0.25)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand((B, 3, max(1, H // 16), max(1, W // 16)), generator=g)
    x = F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)
    x = (x + 0.05 * torch.randn((B, 3, H, W), generator=g)).clamp(0, 1)
    return ((x - 0.4) / 0.25).contiguous()


@functools.lru_cache(maxsize=None)
def experts(E):
    return [O.kaiming_state_dict(100 + e, mean=(0.5 * e, -1.0, 2.0 + e)) for e in range(E)]


@functools.lru_cache(maxsize=None)
def stack(E):
    return ExpertStack(experts(E), "cuda")


def torch_tf32(sd, image):
    """The reference's per-expert route on the device: float32 convolutions under cuDNN's TF32 default."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        with torch.no_grad():
            return O.apply(image.cuda(), {k: v.cuda() for k, v in sd.items()})
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def test_pack_matches_oracle():
    E = 3
    got = stack(E).packed.cpu().numpy()
    want = O.pack(experts(E))
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("hw", [(480, 640), (480, 853), (64, 80)])
def test_accuracy_against_oracle(hw):
    H, W = hw
    E = 3
    img = image_like(1, H, W, seed=H + W)
    out = stack(E).forward(img.cuda())
    torch.cuda.synchronize()
    assert out.shape == (1, E, 3) + prediction_size(H, W)
    for e, sd in enumerate(experts(E)):
        ref = O.forward(img, sd)[0]
        tt = torch_tf32(sd, img)[0].double().cpu()
        ours = out[0, e].double().cpu()
        r_ours = float((ours - ref).norm() / ref.norm())
        r_torch = float((tt - ref).norm() / ref.norm())
        print(f"{H}x{W} expert {e}: stack {r_ours:.3e}, cuDNN TF32 {r_torch:.3e}")
        assert torch.isfinite(ours).all()
        assert r_ours <= 2 * r_torch, (H, W, e, r_ours, r_torch)


def _hist(B, E, active):
    h = torch.zeros(B, E, device="cuda")
    for b, e in active:
        h[b, e] = 3.0
    return h


def test_invariance_active_set_and_batch():
    E, H, W = 4, 120, 168
    st = stack(E)
    img = image_like(1, H, W, seed=5).cuda()
    full = st.forward(img)                         # every pair active
    for e in range(E):
        alone = st.forward(img, _hist(1, E, [(0, e)]))
        other = (e + 1) % E
        pair = st.forward(img, _hist(1, E, [(0, e), (0, other)]))
        assert torch.equal(alone[0, e], full[0, e]) and torch.equal(pair[0, e], full[0, e])
        assert torch.equal(pair[0, other], full[0, other])
        assert not alone[0, other].any()
    imgs = torch.cat([img, image_like(1, H, W, seed=6).cuda(), image_like(1, H, W, seed=7).cuda()])
    for b in range(3):
        batch = torch.cat([imgs[b:b + 1]] * 3)
        batch[(b + 1) % 3] = imgs[(b + 1) % 3]
        out = st.forward(batch.contiguous(), _hist(3, E, [(b, e) for e in range(E)] + [((b + 1) % 3, 1)]))
        single = st.forward(imgs[b:b + 1])
        assert torch.equal(out[b], single[0]), b
    shared = st.forward(img, torch.ones(3, E, device="cuda"))   # one image for every position of the batch
    for b in range(3):
        assert torch.equal(shared[b], full[0])


def test_capture_replays_and_inactive_planes():
    E, H, W = 4, 96, 136
    st = ExpertStack(experts(E), "cuda")      # its own: the capture freezes its workspace
    img = image_like(1, H, W, seed=9).cuda()
    hist = torch.zeros(2, E, device="cuda")
    out = torch.full((2, E, 3) + prediction_size(H, W), float("nan"), device="cuda")
    st.reserve(2, H, W)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        st.forward_async(img, hist, out)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st.forward_async(img, hist, out)
    eager_all = st.forward(img, torch.ones(2, E, device="cuda"))
    with pytest.raises(RuntimeError, match="a captured graph already uses"):
        st.forward(image_like(1, 4 * H, W, seed=1).cuda())   # needs more than the two images reserved
    rng = np.random.default_rng(3)
    prev = None
    for r in range(20):
        h = (rng.random((2, E)) < 0.5).astype(np.float32) * rng.integers(1, 50, (2, E))
        if r % 5 == 0:
            h[:] = 0 if r % 10 == 0 else 1
        hist.copy_(torch.from_numpy(h))
        graph.replay()
        eager = st.forward(img, hist)
        torch.cuda.synchronize()
        assert torch.equal(out, eager), r
        for b in range(2):
            for e in range(E):
                if h[b, e] > 0:
                    assert torch.equal(out[b, e], eager_all[b, e]), (r, b, e)
                else:
                    assert not out[b, e].any(), (r, b, e)   # zero, also where the previous replay wrote it
        prev = h
    assert prev is not None


def test_capture_needs_reserved_workspace():
    E = 2
    st = ExpertStack(experts(E), "cuda")
    img = image_like(1, 64, 64, seed=1).cuda()
    out = torch.empty((1, E, 3, 8, 8), device="cuda")
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="reserve"):
        with torch.cuda.graph(graph):
            st.forward_async(img, None, out)


def test_example_check():
    path = ROOT / "examples" / "test_step_expert_stack_graph_synthetic.py"
    spec = importlib.util.spec_from_file_location("expert_stack_example", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.main(["--images", "4", "--experts", "5", "--check"]) == 0
