"""Each single-image entry point hands the library its scalar tail, shiftX .. subSampling, at the place and in the order of
the prototype in include/esac_b200.h, as Python ints and floats whatever number types the caller passed; the three sharded
calls set the context's hypothesis-shard options for the call and reset them even when it raises.  The library is a stub
here (no context, no device): it records every call."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200.synth import make_scene

HEADER = Path(__file__).resolve().parents[1] / "include" / "esac_b200.h"
E, H, W, M = 2, 8, 10, 4
TAIL_NAMES = ["shiftX", "shiftY", "focalLength", "ppointX", "ppointY", "inlierThreshold", "inlierAlpha", "inlierBeta",
              "maxReproj", "subSampling"]
# numpy, torch and Python numbers of every kind, and what ctypes must receive for them
GIVEN = (np.int64(3), -2, np.float32(525.3), 320, torch.tensor(240.5), 10, np.float64(100.0), 0.5, 100, np.int32(8))
WANT = (3, -2, float(np.float32(525.3)), 320.0, 240.5, 10.0, 100.0, 0.5, 100.0, 8)


def _prototype(name):
    """(C type, parameter name) of each parameter of `name` in the public header."""
    m = re.search(r"\b" + name + r"\((.*?)\);", HEADER.read_text(), re.S)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [tuple(p.rsplit(" ", 1)) for p in params]


class Lib:
    def __init__(self):
        self.calls, self.fail = [], None

    def __getattr__(self, name):
        def entry(*args):
            self.calls.append((name, args))
            if self.fail == name:
                raise RuntimeError("stub failure")
            return 0
        return entry


class Ctx:
    handle, device = None, 0

    def __init__(self):
        self.lib = Lib()

    def check(self, rc):
        assert rc == 0

    def set_stream(self, stream):
        pass

    def set_option(self, key, value):
        self.lib.calls.append(("set_option", (key, value)))


class _cuda:
    """A host tensor that passes for a CUDA one (forward_pack takes CUDA tensors only); the stub reads no memory."""
    __module__ = "torch.stub"
    is_cuda = True

    def __init__(self, t):
        self.t = t

    def __getattr__(self, key):
        return getattr(self.t, key)


@pytest.fixture
def ctx(monkeypatch):
    stub = Ctx()
    monkeypatch.setattr(api, "_pick_ctx", lambda *devices: stub)
    monkeypatch.setattr(api, "_pick_ctx_host", lambda device: stub)
    monkeypatch.setattr(api, "hypotheses_tape_bytes", lambda E, H, W, M: 16)
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda *a, device=None, **k: empty(*a, **k))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: type("Stream", (), {"cuda_stream": 0}))
    return stub


@pytest.fixture(scope="module")
def scene():
    s = make_scene(E=E, H=H, W=W, M=M, seed=0)
    return {"coords": torch.from_numpy(s.coords), "assign": torch.from_numpy(s.assign), "gt": torch.from_numpy(s.gt_pose)}


def _calls(s, tail):
    """Every single-image entry point of api.py with the scalar tail `tail`."""
    grads = torch.zeros_like(s["coords"])
    return {
        "esacb200_forward": lambda: api.forward(s["coords"], s["assign"], torch.zeros(4, 4), *tail),
        "esacb200_backward": lambda: api.backward(s["coords"], grads, s["assign"], s["gt"], 1.0, 100.0, 100.0, *tail),
        "esacb200_backward_sharded": lambda: api.backward_sharded(s["coords"], grads, s["assign"], s["gt"], 1.0, 100.0, 100.0,
                                                                  *tail, lambda phase, values: values, hyp_offset=5),
        "esacb200_backward_sharded_nccl": lambda: api.backward_sharded_nccl(s["coords"], grads, s["assign"], s["gt"], 1.0, 100.0,
                                                                            100.0, *tail, hyp_offset=5, hyp_stride=3),
        "esacb200_forward_sharded": lambda: api.forward_sharded(s["coords"], s["assign"], torch.zeros(4, 4), *tail,
                                                                hyp_offset=5, hyp_stride=3),
        "esacb200_forward_pack": lambda: api.forward_pack(_cuda(s["coords"]), _cuda(s["assign"]), tail, 0,
                                                          _cuda(torch.zeros(M + api.PACK_TAIL, dtype=torch.float64))),
        "esacb200_score_poses": lambda: api.score_poses(s["coords"], s["assign"], np.zeros((M, 6)), *tail),
        "esacb200_hypotheses_forward": lambda: api.hypotheses_forward(s["coords"], s["assign"], *tail),
    }


def test_the_scalar_tail_reaches_the_library_in_header_order(ctx, scene):
    for name, call in _calls(scene, GIVEN).items():
        ctx.lib.calls.clear()
        call()
        (got,) = [args for n, args in ctx.lib.calls if n == name]
        proto = _prototype(name)
        assert len(got) == len(proto), name
        at = [p for _, p in proto].index("shiftX")
        assert [p for _, p in proto[at:at + 10]] == TAIL_NAMES, name
        tail = got[at:at + 10]
        assert tail == WANT, name
        assert [type(v) for v in tail] == [int if t == "int" else float for t, _ in proto[at:at + 10]], name


SHARD_OPTIONS = {"esacb200_backward_sharded": [("hyp_offset", 5)],
                 "esacb200_backward_sharded_nccl": [("hyp_offset", 5), ("hyp_stride", 3)],
                 "esacb200_forward_sharded": [("hyp_offset", 5), ("hyp_stride", 3)]}
RESET = {"hyp_offset": 0, "hyp_stride": 1}


@pytest.mark.parametrize("name", sorted(SHARD_OPTIONS))
@pytest.mark.parametrize("raises", [False, True])
def test_sharded_calls_reset_the_shard_options(ctx, scene, name, raises):
    ctx.lib.fail = name if raises else None
    call = _calls(scene, GIVEN)[name]
    if raises:
        with pytest.raises(RuntimeError, match="stub failure"):
            call()
    else:
        call()
    seen = [(n, args) for n, args in ctx.lib.calls if n in ("set_option", name)]
    options = SHARD_OPTIONS[name]
    want = ([("set_option", o) for o in options] + [(name, seen[len(options)][1])] +
            [("set_option", (k, RESET[k])) for k, _ in options])
    assert seen == want
