"""CUDA path against outputs of the reference's OWN compiled code (tests/golden/ref_*.npz; how they were made:
tests/golden/make_ref_golden.py -- the unmodified esac.cpp on the real OpenCV, single thread, default mt19937 stream).

The fixtures carry every minimal set the reference tried; they are injected (esacb200_inject_cells) so the CUDA path judges
the same candidates in the same order.  Tolerances: 1e-3 deg / 1e-3 cm on the pose and the expected loss to 1e-6 relative
(BASELINE.json).  Gradients: 1e-3 of the largest entry, and class by class (tests/grad_terms.py) -- on the small fixtures
minimal-set, final-inlier and other cells, classed by a cv2 oracle run on the injected sets, each to BAR_SMALL of its own
largest entry; on the 120x160 and 480x640 fixtures the sampled entries outside every contributing minimal set to BAR_SAMPLED of
their own largest entry.  Measured on an H100 SXM (80 GB, 700 W), worst over the fixtures: minimal 2.5e-6, inlier 1.4e-6,
rest 4.3e-6 (ref_clamp_jr_on_12x16 aside: 1.1e-5 and 1.6e-5 of a 2.2e-5 gradient, see BAR_CLAMPED), sampled other entries
6.1e-7; the bars are about 10x that and never looser than 1e-4."""
import ast

import numpy as np
import pytest

import grad_terms as GT
from esac_b200.synth import pose_error
from oracle import esac_oracle as O
from ref_golden_util import REF_GOLD, load, params_of

pytestmark = pytest.mark.gpu

BAR_SMALL = {"minimal": 3e-5, "inlier": 1.5e-5, "rest": 5e-5}   # class-wise bar of the small fixtures
# ref_clamp_jr_on_12x16 clamps path I away on every contributing hypothesis (map units of 1/7000 m): what remains is a score
# term of 2.2e-5 at most, which the GPU meets to 3.5e-10, i.e. 1.1e-5 / 1.6e-5 of the minimal / inlier scale
BAR_CLAMPED = GT.CAP
BAR_SAMPLED = 6e-6     # sampled entries outside the contributing minimal sets of the 120x160 and 480x640 fixtures


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


@pytest.mark.parametrize("path", REF_GOLD, ids=[p.stem for p in REF_GOLD])
def test_forward_and_backward_match_the_compiled_reference(api, path):
    z, coords = load(path)
    params = params_of(z)
    cells = z["cells"]
    T = cells.shape[1]
    # ---- esac.forward ----
    api.inject_cells(cells)
    out = np.zeros((4, 4), np.float32)
    e = api.forward(coords, z["assign"], out, *params)
    hy = api.last_hypotheses()
    st = api.last_stats()
    assert hy["tries"].tolist() == np.minimum(z["tries"], T).tolist()      # same verdict on every candidate set
    assert hy["cells"].tolist() == cells[:, -1].tolist()                    # the accepted sets
    assert np.abs(hy["scores"] - z["oracle_scores"]).max() < 1e-4 * max(1.0, params[6] / 100.0)   # scores scale with alpha
    s = np.sort(z["oracle_scores"])[::-1]
    assert s[0] - s[1] > 1e-3, "fixture has a tie at the top: regenerate with another seed"
    assert e == int(z["expert"]) and st["winner"] == int(z["oracle_winner"])
    assert st["refine_rounds"] == int(z["oracle_rounds"])
    rot, trans = pose_error(out, z["pose"])
    unit = float(ast.literal_eval(str(z["scene_kw"])).get("unit_scale", 1.0))  # map units per metre: 1e-3 cm = 1e-5 m
    assert rot < 1e-3 and trans < 1e-5 * unit, (rot, trans)
    # ---- esac.backward ----
    api.inject_cells(cells)
    g = np.zeros_like(coords)
    w_rot, w_trans, cut = (float(v) for v in z["loss_args"])
    loss = api.backward(coords, g, z["assign"], z["gt_pose"], w_rot, w_trans, cut, *params)
    assert abs(loss - float(z["loss"])) < 1e-6 * max(1.0, abs(float(z["loss"])))
    if "grads" in z.files:
        scale = max(np.abs(z["grads"]).max(), 1e-12)
        assert np.abs(g - z["grads"]).max() / scale < 1e-3
        # classes from the cv2 oracle on the same injected minimal sets
        _, bt = O.backward(coords, np.zeros_like(coords), z["assign"], z["gt_pose"], w_rot, w_trans, cut, *params,
                           injected_cells=cells, trace=True)
        assert [list(map(list, h.cells)) for h in bt.hyps] == cells[:, -1].tolist()
        rep = GT.assert_classwise(g, z["grads"], GT.cell_classes(coords.shape, z["assign"], bt),
                                  BAR_CLAMPED if path.stem == "ref_clamp_jr_on_12x16" else BAR_SMALL, path.stem)
        print(f"{path.stem}: {GT.fmt(rep)}")
        if "unclamped_grad_diff" in z.files and "_off_" not in path.stem:
            # clamp fixtures (esac.cpp:436-437, esac_derivative.h:287): without the `> 10` clamps the gradient would sit this
            # far away (tests/test_oracle.py::test_clamp_fixtures_really_trip_the_clamps), i.e. >= 50 tolerances
            assert float(z["unclamped_grad_diff"]) / scale > 0.05
    else:
        scale = float(z["grad_max"])
        assert abs(np.abs(g).max() - scale) < 1e-3 * scale
        got = g.reshape(-1)[z["grad_idx"]].astype(np.float64)
        assert np.abs(got - z["grad_val"]).max() / scale < 1e-3
        # the sampled entries outside every contributing minimal set, against their own largest entry
        other = ~GT.sampled_classes(z["grad_idx"], g.shape, z["assign"], cells[:, -1], O.softmax(z["oracle_scores"]))
        assert 0 < other.sum() < other.size
        oscale = max(np.abs(z["grad_val"][other]).max(), GT.FLOOR * scale)
        rel = np.abs(got[other] - z["grad_val"][other]).max() / oscale
        print(f"{path.stem}: other {rel:.2e} of {oscale:.2e} ({other.sum()} of {other.size} entries), "
              f"all {np.abs(got - z['grad_val']).max() / scale:.2e} of {scale:.2e}")
        assert rel <= BAR_SAMPLED, (rel, oscale)
        ps = g.astype(np.float64).sum(axis=(2, 3))
        pa = np.abs(g).astype(np.float64).sum(axis=(2, 3))
        assert np.abs(ps - z["grad_plane_sum"]).max() < 1e-3 * max(z["grad_plane_abs"].max(), 1e-12)
        assert np.abs(pa - z["grad_plane_abs"]).max() < 1e-3 * max(z["grad_plane_abs"].max(), 1e-12)
