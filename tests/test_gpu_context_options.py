"""Options set on a context reach the worker contexts of the batched entry points: backward_batch and
hypotheses_forward_batch launch and compute, image by image, what B consecutive single-image calls on the same context do
(run with `-m gpu`)."""
import numpy as np
import pytest

from esac_b200.synth import make_scene

pytestmark = pytest.mark.gpu

W_LOSS = (1.0, 100.0, 100.0)
DEFAULTS = {"sample_waves": 6, "sample_groups": 2, "fixed_seed": 0, "batch_workers": 8}


# The sampling stage launches a fixed number of kernels per wave and per lane, so a worker that ignored the option would
# launch a different number of kernels than the loop.  sample_groups = 1 needs a map on which the default runs two lanes
# (at least 65,536 cells and 64 hypotheses).
@pytest.mark.parametrize("key,value,H,W,M", [("sample_waves", 2, 24, 32, 24), ("sample_groups", 1, 256, 256, 64)])
def test_batched_calls_honour_the_context_options(key, value, H, W, M):
    import torch
    import esac_b200.api as api
    B = 3
    scenes = [make_scene(E=2, H=H, W=W, M=M, sub=8, seed=90 + b) for b in range(B)]
    coords = torch.from_numpy(np.stack([s.coords for s in scenes])).cuda()
    assign = torch.from_numpy(np.stack([s.assign for s in scenes])).cuda()
    gts = torch.from_numpy(np.stack([s.gt_pose for s in scenes])).cuda()
    p = scenes[0].params  # the same camera for every image of one size
    ctx = api.context()
    try:
        ctx.set_option("batch_workers", 1)
        ctx.set_option("fixed_seed", 0)
        ctx.set_option(key, value)

        api.set_seed(17)
        g_loop = torch.zeros_like(coords)
        l_loop, n_loop = [], 0
        for b in range(B):
            l_loop.append(api.backward(coords[b], g_loop[b], assign[b], gts[b], *W_LOSS, *p))
            n_loop += api.last_stats()["kernel_launches"]
        api.set_seed(17)
        g_batch = torch.zeros_like(coords)
        l_batch = api.backward_batch(coords, g_batch, assign, gts, *W_LOSS, *p)
        assert api.last_stats()["kernel_launches"] == n_loop
        assert np.allclose(l_batch, l_loop, rtol=1e-12, atol=0)
        assert torch.equal(g_batch, g_loop)

        api.set_seed(18)
        loop, n_loop = [], 0
        for b in range(B):
            loop.append(api.hypotheses_forward(coords[b], assign[b], *p))
            n_loop += api.last_stats()["kernel_launches"]
        api.set_seed(18)
        scores, poses, contrib, _ = api.hypotheses_forward_batch(coords, assign, *p)
        assert api.last_stats()["kernel_launches"] == n_loop
        for b in range(B):
            assert torch.equal(scores[b], loop[b][0]), b
            assert torch.equal(poses[b], loop[b][1]), b
            assert torch.equal(contrib[b], loop[b][2]), b
    finally:
        for k in (key, "fixed_seed", "batch_workers"):
            ctx.set_option(k, DEFAULTS[k])
