"""Both forms of the scoring kernel's cell tail against the float64 reference (oracle/score_fp64.py).

With k1 = beta log2(e) > 0 and a clamp exponent k1 maxReproj - beta tau log2(e) - 32 <= 63 the kernel folds k1 into the
pose rows and pixel offsets and takes one reciprocal per pair of cells; otherwise (here maxReproj = 300, or beta <= 0) it
keeps one reciprocal per cell.  The bench parameters (tau 10, beta 0.5, maxReproj 100) take the folded form."""
import numpy as np
import pytest

from esac_b200.synth import make_scene
from oracle import score_fp64
from test_gpu_score_shapes import _dense_poses, score_forced

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-4


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


@pytest.mark.parametrize("max_reproj,beta,folded", [(100.0, 0.5, True), (300.0, 0.5, False), (100.0, 0.0, False),
                                                    (100.0, -0.05, False)])
@pytest.mark.parametrize("H,W,sub", [(120, 160, 4), (61, 81, 3)])
def test_cell_tail_forms_match_the_reference(api, max_reproj, beta, folded, H, W, sub):
    import torch
    sc = make_scene(E=3, H=H, W=W, M=36, sub=sub, seed=41, shiftX=3, shiftY=-5)
    poses = _dense_poses(sc, np.random.default_rng(41), len(sc.assign))
    params = list(sc.params)
    params[7], params[8] = beta, max_reproj
    k1 = np.float32(beta) * np.float32(1.4426950408889634)
    k0 = -np.float32(beta) * np.float32(sc.tau) * np.float32(1.4426950408889634)
    assert (k1 >= 1e-3 and float(k1) * max_reproj + float(k0) - 32 <= 63) == folded
    ref, _ = score_fp64.score(sc.coords, sc.assign, poses, *params)
    t = torch.from_numpy(sc.coords).cuda()
    a = torch.from_numpy(sc.assign).cuda()
    for ppt in (2, 4, 8):
        got = score_forced(api, t, a, poses, params, ppt, 16)
        assert np.abs(got - ref).max() < SCORE_TOL, (ppt, np.abs(got - ref).max())
