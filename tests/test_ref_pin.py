"""Pins the oracle to the reference's OWN compiled code.

oracle/_ref/esac_ref is the unmodified code/esac/{esac.cpp,thread_rand.cpp} of vislearn/esac (+ its headers) compiled
against oracle/ref_shim/opencv2/opencv.hpp, whose solvePnP / projectPoints / Rodrigues / Mat::inv are executed by the real
OpenCV inside the cv2 wheel (oracle/build_ref.py).  With one OpenMP thread the reference consumes one std::mt19937 stream
in a fixed order; oracle.esac_oracle.ThreadRandStream reproduces that stream, so both see identical minimal sets and every
output of esac_forward / esac_backward can be compared.  What the compiled reference returned for the calls below is stored
in tests/golden/pin/ref_pin.npz (tests/golden/make_ref_pin.py); the two tests of the compiled stand-in itself are skipped
where oracle/_ref is not built.
"""
from pathlib import Path

import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error
from oracle import esac_oracle as O
from oracle.build_ref import load_ref

torch = pytest.importorskip("torch")
GOLD = Path(__file__).resolve().parent / "golden" / "pin" / "ref_pin.npz"


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def ref():
    mod = load_ref()
    if mod is None:
        pytest.skip("oracle/_ref is not built and no readable reference checkout was found (oracle/build_ref.py)")
    mod.set_num_threads(1)
    mod.set_native_project(False)
    return mod


IRAND_MAX = (79, 59, 639, 479, 2, 3_000_000_000 // 2, 7)


def test_thread_rand_stream_is_the_references(gold):
    """thread_rand.cpp:34-43,68-71 on generator 0 == ThreadRandStream (mt19937 + libstdc++ uniform_int_distribution)."""
    mt = O.ThreadRandStream(1305)
    for exc_max, a in zip(IRAND_MAX, gold["irand_1305"].tolist()):
        b = [mt.irand(0, exc_max) for _ in range(300)]
        assert a == b
        assert max(a) <= exc_max - 1 and min(a) >= 0
    mt = O.ThreadRandStream(77)
    assert gold["irand_77"].tolist() == [mt.irand(3, 11) for _ in range(50)]


CASES = {
    "c1_60x80": dict(E=1, H=60, W=80, M=64, sub=8, seed=3),
    "ensemble3_shift": dict(E=3, H=30, W=40, M=32, sub=8, seed=3, shiftX=3, shiftY=-2),
    "world_scale": dict(E=2, H=24, W=32, M=24, sub=8, seed=3, outdoor=True, world_offset=700.0),
    "portrait_odd": dict(E=2, H=40, W=27, M=24, sub=8, seed=4),
}


@pytest.mark.parametrize("name", list(CASES))
def test_forward_and_backward_equal_the_compiled_reference(gold, name):
    sc = make_scene(**CASES[name])
    # forward: esac.cpp:64-190
    mine = np.zeros((4, 4), np.float32)
    e_or = O.forward(sc.coords, sc.assign, mine, *sc.params, mt=O.ThreadRandStream(1305))
    assert int(gold[f"{name}_expert"]) == e_or
    assert np.abs(gold[f"{name}_pose"] - mine).max() <= 1e-6  # observed: bit-identical
    # backward: esac.cpp:213-511 (accumulates into the caller's tensor: start from a non-zero one)
    l_ref, g_ref = float(gold[f"{name}_loss"]), gold[f"{name}_grads"]
    g_or = np.full(sc.coords.shape, 0.25, np.float32)
    l_or = O.backward(sc.coords, g_or, sc.assign, sc.gt_pose, 1.0, 100.0, 100.0, *sc.params, mt=O.ThreadRandStream(1305))
    assert abs(l_ref - l_or) <= 1e-9 * max(1.0, abs(l_ref))
    scale = np.abs(g_or - 0.25).max()
    assert scale > 0
    assert np.abs(g_ref - g_or).max() <= 1e-6 * scale  # observed: <= 3e-9


CUT_SCENE = dict(E=2, H=24, W=32, M=24, sub=8, seed=9)
CUT_CASES = ((1.0, 100.0, 5.0), (0.5, 10.0, 1000.0))


def test_loss_cut_and_weights_equal_the_compiled_reference(gold):
    """The cut branch (esac_loss.h:78-80 vs :133-137,202-203 -- the sqrt(cut*loss) / 0.5/sqrt(loss) mismatch) and
    non-default weights, on a scene whose poses are far from a deliberately wrong ground truth."""
    sc = make_scene(**CUT_SCENE)
    gt = sc.gt_pose.copy()
    gt[:3, 3] += np.array([3.0, -2.0, 1.0], np.float32)
    for i, (w_rot, w_trans, cut) in enumerate(CUT_CASES):
        l_ref, g_ref = float(gold[f"cut{i}_loss"]), gold[f"cut{i}_grads"]
        g_or = np.zeros_like(sc.coords)
        l_or = O.backward(sc.coords, g_or, sc.assign, gt, w_rot, w_trans, cut, *sc.params, mt=O.ThreadRandStream(1305))
        assert abs(l_ref - l_or) <= 1e-9 * max(1.0, abs(l_ref))
        assert np.abs(g_ref - g_or).max() <= 1e-6 * max(np.abs(g_or).max(), 1e-30)


# the fixtures of tests/golden/make_ref_golden.py away from the reference's default hyperparameters: each stores its
# make_scene arguments, its (shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub) and its loss arguments
PARAM_FIXTURES = ("ref_params_tight_30x40", "ref_params_clamp_30x40", "ref_params_subpx_24x32")


def _param_case(name):
    """(fixture, scene regenerated from its make_scene arguments, parameters, loss arguments)."""
    import ast
    from ref_golden_util import params_of
    z = np.load(GOLD.parents[1] / f"{name}.npz")
    sc = make_scene(**ast.literal_eval(str(z["scene_kw"])))
    assert np.array_equal(z["coords"], sc.coords) and np.array_equal(z["assign"], sc.assign)
    return z, sc, params_of(z), tuple(float(v) for v in z["loss_args"])


def test_parameter_fixtures_leave_the_defaults():
    """tau 2 / beta 2 / alpha 50 with the loss (0.5, 30, 5); tau 40 above maxReproj 30, beta 0.1, alpha 400; tau 0.6 px."""
    got = {name: (_param_case(name)[2][5:9], _param_case(name)[3]) for name in PARAM_FIXTURES}
    assert got == {"ref_params_tight_30x40": ((2.0, 50.0, 2.0, 100.0), (0.5, 30.0, 5.0)),
                   "ref_params_clamp_30x40": ((40.0, 400.0, 0.1, 30.0), (1.0, 100.0, 100.0)),
                   "ref_params_subpx_24x32": ((0.6, 100.0, 0.5, 100.0), (1.0, 100.0, 100.0))}


@pytest.mark.parametrize("name", PARAM_FIXTURES)
def test_oracle_equals_the_compiled_reference_away_from_the_defaults(name):
    """What the compiled reference returned is the fixture; the oracle must return it too, on the scene regenerated from the
    fixture's make_scene arguments."""
    z, sc, params, loss_args = _param_case(name)
    mine = np.zeros((4, 4), np.float32)
    assert O.forward(sc.coords, sc.assign, mine, *params, mt=O.ThreadRandStream(1305)) == int(z["expert"])
    assert np.abs(z["pose"] - mine).max() <= 1e-6
    g_or = np.zeros_like(sc.coords)
    l_or = O.backward(sc.coords, g_or, sc.assign, sc.gt_pose, *loss_args, *params, mt=O.ThreadRandStream(1305))
    assert abs(float(z["loss"]) - l_or) <= 1e-9 * max(1.0, abs(float(z["loss"])))
    assert np.abs(z["grads"] - g_or).max() <= 1e-6 * np.abs(g_or).max()


@pytest.mark.parametrize("name", PARAM_FIXTURES)
def test_compiled_reference_away_from_the_defaults_still_gives_the_fixture(ref, name):
    z, sc, params, loss_args = _param_case(name)
    co, asg = torch.from_numpy(sc.coords), torch.from_numpy(sc.assign)
    ref.force_init(1305)
    pose = torch.zeros(4, 4)
    assert ref.forward(co, asg, pose, *params) == int(z["expert"])
    assert np.array_equal(pose.numpy(), z["pose"])
    ref.force_init(1305)
    g = torch.zeros(sc.coords.shape)
    loss = ref.backward(co, g, asg, torch.from_numpy(sc.gt_pose), *loss_args, *params)
    assert loss == float(z["loss"]) and np.array_equal(g.numpy(), z["grads"])


PERSIST_SCENE = dict(E=1, H=24, W=32, M=16, sub=8, seed=11)


def test_stream_state_persists_across_calls(gold):
    """thread_rand.cpp:4-5: static generators -- a second call continues the stream; so does the oracle's object."""
    sc = make_scene(**PERSIST_SCENE)
    mt = O.ThreadRandStream(1305)
    for out in gold["persist_poses"]:
        mine = np.zeros((4, 4), np.float32)
        O.forward(sc.coords, sc.assign, mine, *sc.params, mt=mt)
        assert np.abs(out - mine).max() <= 1e-6


def test_native_projection_of_the_shim_is_bit_identical(ref):
    """The timing-only fast path of the shim (projectPoints without Jacobian as a native loop) changes nothing."""
    sc = make_scene(E=2, H=30, W=40, M=32, sub=8, seed=5, outdoor=True, world_offset=300.0)
    co, asg = torch.from_numpy(sc.coords), torch.from_numpy(sc.assign)
    outs = []
    for native in (False, True):
        ref.set_native_project(native)
        ref.force_init(1305)
        out = torch.zeros(4, 4)
        e = ref.forward(co, asg, out, *sc.params)
        outs.append((e, out.numpy().copy()))
    ref.set_native_project(False)
    assert outs[0][0] == outs[1][0] and np.array_equal(outs[0][1], outs[1][1])


def test_openmp_threads_do_not_deadlock_and_find_the_pose(ref):
    """More than one OpenMP thread: the sample stream is schedule-dependent (not comparable), the estimate is not."""
    sc = make_scene(E=2, H=30, W=40, M=32, sub=8, seed=6, noise=0.0, outlier_frac=0.2)
    ref.set_num_threads(4)
    try:
        ref.force_init(1305)
        out = torch.zeros(4, 4)
        e = ref.forward(torch.from_numpy(sc.coords), torch.from_numpy(sc.assign), out, *sc.params)
    finally:
        ref.set_num_threads(1)
    rot, trans = pose_error(out.numpy(), sc.gt_pose)
    assert e == sc.gt_expert and rot < 0.05 and trans < 0.01
