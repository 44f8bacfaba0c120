"""Bad argument lists of the C entry points: each returns ESACB200_ERR_ARG with one exact message, whatever else is wrong
with the call, because every entry point checks its arguments in one fixed order (run with `-m gpu`).  A failing
forward_pack still clears the statistics, the last-call record and the injected cells, like any call that began.

The calls go through ctypes with the library's own argument lists; pointers the checks reject first are never read."""
import ctypes as C

import numpy as np
import pytest

from esac_b200.synth import make_scene

pytestmark = pytest.mark.gpu

E, H, W, M = 2, 30, 40, 32
W_LOSS = (1.0, 100.0, 100.0)
ERR_ARG = -2
TOO_SMALL = "map 2x2 too small to draw 4 distinct cells from [0,W-2]x[0,H-2]"


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    ctx = api.context()
    ctx.set_stream(0)
    ctx.set_option("fixed_seed", 1)
    return api


@pytest.fixture(scope="module")
def sc():
    return make_scene(E=E, H=H, W=W, M=M, sub=8, seed=3)


@pytest.fixture(autouse=True)
def no_injected_cells(api):
    api.context().inject_cells(None)
    yield
    api.context().inject_cells(None)


def _call(api, name, *args):
    """esacb200_<name>(ctx, *args): the status and the context's message."""
    ctx = api.context()
    rc = getattr(ctx.lib, "esacb200_" + name)(ctx.handle, *args)
    return rc, ctx.lib.esacb200_last_error(ctx.handle).decode()


_ALIVE = []  # every array whose address a test hands to the library, kept for the session


def _ptr(a):
    _ALIVE.append(a)
    return a.ctypes.data


def _ptrs(*values):
    return (C.c_void_p * len(values))(*values)


def _ints(*values):
    return (C.c_int * len(values))(*values)


def _floats(*values):
    return (C.c_float * len(values))(*values)


def _inject(api, m):
    api.context().inject_cells(np.ones((m, 1, 4, 2), np.int32))


def _single(sc, coords, E, H, W, M, tail=None):
    """The argument lists of the single-image entry points on host arrays (sizes as given, not those of the arrays)."""
    c, a = (_ptr(sc.coords), _ptr(sc.assign)) if coords else (None, None)
    out, grads, gt = np.zeros((4, 4), np.float32), np.zeros_like(sc.coords), sc.gt_pose
    tail = tail or sc.params
    loss = C.c_double()
    return {
        "forward": (c, E, H, W, a, 1, M, _ptr(out) if coords else None, *tail, None),
        "backward": (c, _ptr(grads) if coords else None, E, H, W, a, 1, M, _ptr(gt) if coords else None, *W_LOSS, *tail,
                     C.byref(loss)),
        "score_poses": (c, E, H, W, a, 1, M, _ptr(np.zeros((max(M, 1), 6))) if coords else None, *tail,
                        _ptr(np.zeros(max(M, 1))) if coords else None),
    }


def test_a_null_pointer_is_reported_before_bad_sizes(api, sc):
    for name, args in _single(sc, False, 0, 2, 2, 0).items():
        assert _call(api, name, *args) == (ERR_ARG, "null pointer argument"), name
    tail = sc.params
    assert _call(api, "hypotheses_forward", None, 0, 2, 2, None, 1, 0, *tail, None, 0, None, None, None) == \
        (ERR_ARG, "null pointer argument")
    assert _call(api, "backward_sharded", None, None, 0, 2, 2, None, 1, 0, None, *W_LOSS, *tail, api.EXCHANGE_FN(), None, None) == \
        (ERR_ARG, "exchange callback is null")
    assert _call(api, "forward_pack", None, 0, 2, 2, None, 1, 4, 4, *tail, 0, None) == (ERR_ARG, "null pointer argument")
    assert _call(api, "forward_ragged", 0, None, None, None, 0, None, 1, 0, None, None, None, None, None, None, *tail[5:],
                 None) == (ERR_ARG, "null pointer argument or empty batch")
    for name, n in (("forward_async", 7), ("backward_async", 8)):
        head = (0, None, 0, 2, 2, None, 1, 0) if name == "forward_async" else (0, None, None, 0, 2, 2, None, 1, 0, None, *W_LOSS)
        rest = (None, None, None) if name == "forward_async" else (None, None)
        assert _call(api, name, *head, None, None, *tail[5:], *rest) == (ERR_ARG, f"{name}: empty batch (B=0)"), name


def test_empty_sizes(api, sc):
    for name, args in _single(sc, True, 0, H, W, M).items():
        assert _call(api, name, *args) == (ERR_ARG, f"empty tensor (E=0 H={H} W={W} M={M})"), name
    for name, args in _single(sc, True, E, H, W, 0).items():
        assert _call(api, name, *args) == (ERR_ARG, f"empty tensor (E={E} H={H} W={W} M=0)"), name
    # the stream-ordered calls check the sizes before their pointers
    assert _call(api, "forward_async", 1, None, 0, H, W, None, 1, M, None, None, *sc.params[5:], None, None, None) == \
        (ERR_ARG, f"empty tensor (E=0 H={H} W={W} M={M})")
    # a shard without hypotheses is legal
    import torch
    pack = torch.zeros(1 + 21, dtype=torch.float64, device="cuda")
    assert _call(api, "forward_pack", None, E, H, W, None, 1, 0, 1, *sc.params, 0, pack.data_ptr())[0] == 0
    torch.cuda.synchronize()


def test_a_map_too_small_to_draw_from(api, sc):
    for name, args in _single(sc, True, E, 2, 2, M).items():
        if name != "score_poses":  # which draws nothing: a 2x2 map is legal there
            assert _call(api, name, *args) == (ERR_ARG, TOO_SMALL), name
    tape = np.zeros(64, np.uint8)
    assert _call(api, "hypotheses_forward", _ptr(sc.coords), E, 2, 2, _ptr(sc.assign), 1, M, *sc.params, _ptr(tape), 64,
                 _ptr(np.zeros(M)), _ptr(np.zeros((M, 6))), _ptr(np.zeros(M, np.uint8))) == (ERR_ARG, TOO_SMALL)
    assert _call(api, "forward_async", 1, None, E, 2, 2, None, 1, M, None, None, *sc.params[5:], None, None, None) == \
        (ERR_ARG, TOO_SMALL)


def test_injected_cells_of_another_m(api, sc):
    _inject(api, 3)
    for name in ("forward", "backward"):
        assert _call(api, name, *_single(sc, True, E, H, W, M)[name]) == \
            (ERR_ARG, f"injected cells are for M=3, call has M={M}"), name
    tape = np.zeros(64, np.uint8)
    assert _call(api, "hypotheses_forward", _ptr(sc.coords), E, H, W, _ptr(sc.assign), 1, M, *sc.params, _ptr(tape), 64,
                 _ptr(np.zeros(M)), _ptr(np.zeros((M, 6))), _ptr(np.zeros(M, np.uint8))) == \
        (ERR_ARG, f"injected cells are for M=3, call has M={M}")


@pytest.mark.parametrize("bad", [(W, 0), (0, H), (-1, 0), (0, -1)])
def test_injected_cells_outside_the_map(api, sc, bad):
    """The sampling kernels read coords at every injected cell unchecked: a set with one cell outside [0,W-1]x[0,H-1] is
    refused before anything launches, on every entry point that draws injected cells."""
    cells = np.zeros((M, 1, 4, 2), np.int32)
    cells[:, 0] = [[0, 0], [W - 1, 0], [0, H - 1], [W - 1, H - 1]]
    cells[M // 2, 0, 3] = bad
    api.context().inject_cells(cells)
    xs, ys = cells[..., 0], cells[..., 1]
    msg = f"injected cells span x {xs.min()}..{xs.max()}, y {ys.min()}..{ys.max()}: outside the {W}x{H} map"
    for name in ("forward", "backward"):
        assert _call(api, name, *_single(sc, True, E, H, W, M)[name]) == (ERR_ARG, msg), name
    tape = np.zeros(64, np.uint8)
    assert _call(api, "hypotheses_forward", _ptr(sc.coords), E, H, W, _ptr(sc.assign), 1, M, *sc.params, _ptr(tape), 64,
                 _ptr(np.zeros(M)), _ptr(np.zeros((M, 6))), _ptr(np.zeros(M, np.uint8))) == (ERR_ARG, msg)


def _ragged(sc, hs, ws, tapes=None, tape_bytes=None):
    """The argument lists of the ragged entry points for len(hs) images (host arrays, never read by a failing check)."""
    B = len(hs)
    coords = _ptrs(*[_ptr(sc.coords)] * B)
    grads = _ptrs(*[_ptr(np.zeros_like(sc.coords)) for _ in range(B)])
    assign = np.stack([sc.assign] * B)
    gts = np.stack([sc.gt_pose] * B)
    cams = (_ints(*[0] * B), _ints(*[0] * B), _floats(*[sc.f] * B), _floats(*[sc.ppx] * B), _floats(*[sc.ppy] * B))
    thr = sc.params[5:]
    tapes = tapes or _ptrs(*[_ptr(np.zeros(16, np.uint8))] * B)
    tape_bytes = tape_bytes or (C.c_size_t * B)(*[1 << 30] * B)
    return {
        "forward_ragged": (B, coords, _ints(*hs), _ints(*ws), E, _ptr(assign), 1, M, _ptr(np.zeros((B, 4, 4), np.float32)), *cams,
                           *thr, None),
        "backward_ragged": (B, coords, grads, _ints(*hs), _ints(*ws), E, _ptr(assign), 1, M, _ptr(gts), *W_LOSS, *cams, *thr,
                            _ptr(np.zeros(B))),
        "hypotheses_forward_ragged": (B, coords, _ints(*hs), _ints(*ws), E, _ptr(assign), 1, M, *cams, *thr, tapes, tape_bytes,
                                      _ptr(np.zeros((B, M))), _ptr(np.zeros((B, M, 6))), _ptr(np.zeros((B, M), np.uint8))),
        "hypotheses_backward_ragged": (B, tapes, coords, grads, _ints(*hs), _ints(*ws), E, None, None),
    }


def test_a_ragged_batch_whose_third_image_is_too_small(api, sc):
    for name, args in _ragged(sc, [H, H, 2], [W, W, 2]).items():
        assert _call(api, name, *args) == (ERR_ARG, "image 2: " + TOO_SMALL), name
    cams = (None, None, _floats(*[sc.f] * 3), _floats(*[sc.ppx] * 3), _floats(*[sc.ppy] * 3))
    assert _call(api, "backward_batch_cameras", 3, _ptr(sc.coords), _ptr(np.zeros_like(sc.coords)), E, 2, 2, _ptr(sc.assign), 0,
                 M, _ptr(np.stack([sc.gt_pose] * 3)), *W_LOSS, *cams, *sc.params[5:], None) == (ERR_ARG, "image 0: " + TOO_SMALL)


def test_injected_cells_on_a_ragged_call(api, sc):
    _inject(api, M)
    for name, args in _ragged(sc, [H, H, 2], [W, W, 2]).items():
        if name == "forward_ragged":
            continue  # draws: clears the injected cells instead
        assert _call(api, name, *args) == (ERR_ARG, "injected cells are a single-image test hook"), name


def test_a_short_or_misaligned_tape(api, sc):
    import torch
    need = api.hypotheses_tape_bytes(E, H, W, M)
    buf = torch.zeros(2 * need + 256, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    outs = (_ptr(np.zeros(M)), _ptr(np.zeros((M, 6))), _ptr(np.zeros(M, np.uint8)))
    single = (_ptr(sc.coords), E, H, W, _ptr(sc.assign), 1, M, *sc.params)
    assert _call(api, "hypotheses_forward", *single, base, need - 1, *outs) == \
        (ERR_ARG, f"tape holds {need - 1} bytes, this call needs {need}")
    assert _call(api, "hypotheses_forward", *single, base + 8, need, *outs) == \
        (ERR_ARG, "tape must be 16-byte aligned device memory")
    host = np.zeros(need + 16, np.uint8)
    assert _call(api, "hypotheses_forward", *single, _ptr(host), need, *outs) == \
        (ERR_ARG, "tape must be 16-byte aligned device memory")
    second = base + need + 128 - (need + 128) % 16
    cases = [((base, second), (need, need - 1), f"image 1: tape holds {need - 1} bytes, this call needs {need}"),
             ((base, second + 8), (need, need), "image 1: tape must be 16-byte aligned device memory"),
             ((base, None), (need, need), "image 1: tape is null")]
    for tapes, sizes, want in cases:
        args = _ragged(sc, [H, H], [W, W], _ptrs(*tapes), (C.c_size_t * 2)(*sizes))["hypotheses_forward_ragged"]
        assert _call(api, "hypotheses_forward_ragged", *args) == (ERR_ARG, want), want


def test_forward_pack_with_bad_sizes_clears_what_the_last_call_left(api, sc):
    import torch
    coords = torch.from_numpy(sc.coords).cuda()
    assign = torch.from_numpy(sc.assign).cuda()
    pack = torch.zeros(M + 21, dtype=torch.float64, device="cuda")
    ctx = api.context()

    def forward():
        return _call(api, "forward", *_single(sc, True, E, H, W, M)["forward"])

    def get_hypotheses():
        rows = np.zeros((M, 6))
        rc = ctx.lib.esacb200_get_hypotheses(ctx.handle, _ptr(rows), None, None, None, None, None, None)
        return rc, ctx.lib.esacb200_last_error(ctx.handle).decode()

    # M_pad is checked before the call begins: what the last call left stays
    assert forward() == (0, "")
    _inject(api, 3)
    assert _call(api, "forward_pack", coords.data_ptr(), E, H, W, assign.data_ptr(), 1, M, 1, *sc.params, 0,
                 pack.data_ptr()) == (ERR_ARG, f"M_pad (1) must be >= M ({M}) and >= 1")
    assert ctx.stats()["M"] == M and get_hypotheses()[0] == 0
    # bad sizes: the call began, so the statistics, the last-call record and the injected cells are gone
    assert _call(api, "forward_pack", coords.data_ptr(), 0, H, W, assign.data_ptr(), 1, M, M, *sc.params, 0,
                 pack.data_ptr()) == (ERR_ARG, f"empty tensor (E=0 H={H} W={W} M={M})")
    stats = ctx.stats()
    assert stats["M"] == 0 and stats["kernel_launches"] == 0
    assert get_hypotheses() == (ERR_ARG, "the last call on this context left no hypotheses")
    assert forward() == (0, "")  # no injected cells of M=3 left to refuse it
    torch.cuda.synchronize()
