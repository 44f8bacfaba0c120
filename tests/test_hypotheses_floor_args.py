"""The hypotheses node's probability floor without a GPU: every Python entry point refuses a floor that is NaN, outside
[0, 1] or not a number before any context exists (so before the library is loaded), and accepts the bounds."""
import math

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import autograd
from esac_b200.synth import make_scene

BAD = [(math.nan, "must lie in"), (-0.1, "must lie in"), (1.5, "must lie in"), ("0.5", "must be a number"),
       (None, "must be a number"), (True, "must be a number")]


@pytest.fixture(scope="module")
def sc():
    return make_scene(E=2, H=8, W=10, M=6)


def _async_args(sc):
    coords = torch.from_numpy(sc.coords)
    M = sc.assign.shape[0]
    return (coords, torch.from_numpy(sc.assign), torch.zeros(2, dtype=torch.int32), torch.tensor([sc.f, sc.ppx, sc.ppy]),
            sc.tau, sc.alpha, sc.beta, sc.max_reproj, sc.sub), M


def _calls(sc):
    """(name, call(min_prob)) of every Python entry point that takes the floor, on CPU inputs."""
    coords, assign = sc.coords, sc.assign
    batch = torch.from_numpy(np.stack([coords, coords]))
    batch_assign = torch.from_numpy(np.stack([assign, assign]))
    aargs, M = _async_args(sc)
    tapes = torch.zeros(api.hypotheses_tape_stride(2, 8, 10, M), dtype=torch.uint8)

    def api_async(m):
        api.hypotheses_forward_async(*aargs, tapes, torch.zeros(M, dtype=torch.float64), torch.zeros(M, 6, dtype=torch.float64),
                                     torch.zeros(M, dtype=torch.bool), torch.zeros((), dtype=torch.int32), minProb=m)

    return [
        ("hypotheses_forward", lambda m: api.hypotheses_forward(coords, assign, *sc.params, minProb=m)),
        ("hypotheses_forward_batch", lambda m: api.hypotheses_forward_batch(batch, batch_assign, *sc.params, minProb=m)),
        ("hypotheses_forward_async", api_async),
        ("esac_hypotheses", lambda m: autograd.esac_hypotheses(torch.from_numpy(coords), torch.from_numpy(assign), *sc.params,
                                                               min_prob=m)),
        ("esac_hypotheses_batch", lambda m: autograd.esac_hypotheses_batch(batch, batch_assign, *sc.params, min_prob=m)),
        ("esac_hypotheses_async", lambda m: autograd.esac_hypotheses_async(*aargs, min_prob=m)),
    ]


@pytest.mark.parametrize("library", [False, True], ids=["no_library", "library"])
@pytest.mark.parametrize("bad,match", BAD, ids=["nan", "negative", "above_one", "string", "none", "bool"])
def test_bad_floor_raises_before_any_context(sc, bad, match, library, monkeypatch):
    """library=False: loading the library or taking a context fails the test, so the check comes first."""
    if not library:
        def no_context(*a, **k):
            raise AssertionError("a context was requested before the floor was checked")
        monkeypatch.setattr(api, "load_library", no_context)
        monkeypatch.setattr(api, "context", no_context)
        monkeypatch.setattr(api, "_pick_ctx", no_context)
        monkeypatch.setattr(api, "hypotheses_tape_stride", lambda *a: 1 << 20)
    for name, call in _calls(sc):
        with pytest.raises(RuntimeError, match=f"{name}: (minProb|min_prob) {match}"):
            call(bad)


def test_floor_check_accepts_the_closed_interval():
    for v in (0, 0.0, 1e-300, 1e-3, np.float32(0.5), np.float64(1.0), 1):
        assert api._min_prob(v, "x") == float(v)
    assert api.PROB_THRESH == 1e-3
