"""GPU tests of the 16-bit expert losses (api.reproj_loss_amp / coord_loss_amp, their _async forms and the 16-bit autograd
nodes behind autograd.reproj_loss / coord_loss / reproj_loss_async / coord_loss_async).

For a float16 / bfloat16 prediction p and q = p.float(): every loss is bitwise the float32 call's on q taken on the same
load path (aligned maps against aligned maps, maps one element off against maps one element off), every gradient is
bitwise (g32 * s).to(p.dtype) with g32 the float32 call's gradient on q, and the nodes give the float32 loss and the p.grad
of the p.float() route, eagerly, replayed from a CUDA graph and inside autocast training steps (run with `-m gpu`)."""
import numpy as np
import pytest

from orientations import cam_to_world, uniform_rotations

pytestmark = pytest.mark.gpu

CUT, SUB = 10.0, 8
DTYPES = ["float16", "bfloat16"]


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def api():
    """The module's own context, so that the stream-ordered workspace here has seen only these tests."""
    import esac_b200.api as api
    saved = api._contexts.get(0)
    ctx = api.Context(0)
    api._contexts[0] = ctx
    try:
        yield api
    finally:
        import torch
        torch.cuda.synchronize()
        if saved is not None:
            api._contexts[0] = saved
        else:
            api._contexts.pop(0, None)
        ctx.close()


def _dt(torch, name):
    return getattr(torch, name)


def _place(torch, x, dtype, offset):
    """A copy of x in dtype, `offset` elements past a fresh allocation (offset 1: off the vector path's alignment)."""
    buf = torch.empty(x.numel() + offset, dtype=dtype, device=x.device)
    v = buf[offset:].view(x.shape)
    v.copy_(x)
    return v


def _form(xs, ragged):
    return list(xs) if ragged else xs[0]


def _bitwise(torch, a, b, what=""):
    """a and b hold the same bits, NaN matching any NaN (torch's cast and cvt.rn give different NaN payloads)."""
    a, b = (list(a), list(b)) if isinstance(a, (list, tuple)) else ([a], [b])
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.shape == y.shape, what
        nx, ny = torch.isnan(x), torch.isnan(y)
        assert torch.equal(nx, ny), what
        bits = torch.int16 if x.element_size() == 2 else torch.int32
        xb, yb = x.masked_fill(nx, 0).view(bits), y.masked_fill(ny, 0).view(bits)
        bad = (xb != yb).nonzero()
        assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} differ, first at {bad[0].tolist()}: {x[tuple(bad[0])]} vs {y[tuple(bad[0])]}"


def _expected(torch, g32, s, dtype):
    """(g32 * s).to(dtype): autograd's gradient of p through p.float() for an upstream gradient s."""
    g32 = g32 if isinstance(g32, (list, tuple)) else [g32]
    return [(g * s if s is not None else g).to(dtype) for g in g32]


def _scales(torch, B):
    gen = torch.Generator().manual_seed(B)
    return [None, torch.full((1,), 65536.0 / B, device="cuda"),
            (torch.rand((), generator=gen) * 1000 + 1e-3).cuda().reshape(())]


def _poke(torch, p):
    """NaN and infinite predictions in image 0."""
    p[0, 0, 0] = float("nan")
    p[1, 1, 2] = float("inf")
    p[2, 2, 3] = float("-inf")


# ------------------------------------------------------------------------------------------------
# data
def _reproj_data(torch, shapes, seed):
    """World coordinates in front of each camera (a few behind it), camera->world ground truths, pads and cameras."""
    rng = np.random.default_rng(seed)
    rots = uniform_rotations(len(shapes), seed)
    preds, gts = [], []
    for (H, W), R in zip(shapes, rots):
        T = cam_to_world(R, rng.uniform(-2.0, 2.0, 3)).astype(np.float64)
        z = rng.uniform(1.0, 6.0, (H, W))
        z[rng.random((H, W)) < 0.03] = -0.5
        x, y = (rng.random((H, W)) - 0.5) * z, (rng.random((H, W)) - 0.5) * z
        world = (T @ np.stack([x, y, z, np.ones_like(z)]).reshape(4, -1))[:3].reshape(3, H, W)
        preds.append(torch.from_numpy(world.astype(np.float32)).cuda())
        gts.append(T.astype(np.float32))
    shifts = torch.from_numpy(rng.integers(-4, 5, (len(shapes), 2)).astype(np.int32)).cuda()
    cams = torch.from_numpy(np.array([[rng.uniform(400, 600), W * SUB / 2 + rng.uniform(-5, 5), H * SUB / 2 + rng.uniform(-5, 5)]
                                      for H, W in shapes], np.float32)).cuda()
    return preds, torch.from_numpy(np.stack(gts)).cuda(), shifts, cams


def _coord_data(torch, pshapes, gshapes, seed):
    """Ground truths with invalid (all-zero) cells and predictions near them, some beyond the cut."""
    rng = np.random.default_rng(seed)
    preds, gts = [], []
    for (Hp, Wp), (Hg, Wg) in zip(pshapes, gshapes):
        gt = rng.uniform(-5, 5, (3, Hg, Wg)).astype(np.float32)
        gt[:, rng.random((Hg, Wg)) < 0.1] = 0.0
        p = rng.uniform(-5, 5, (3, Hp, Wp))
        H, W = min(Hp, Hg), min(Wp, Wg)
        p[:, :H, :W] = gt[:, :H, :W] + rng.standard_normal((3, H, W)) * rng.choice([0.5, 30.0], (1, H, W), p=[0.8, 0.2])
        preds.append(torch.from_numpy(p.astype(np.float32)).cuda())
        gts.append(torch.from_numpy(gt).cuda())
    return preds, gts


def _stack_or_list(torch, xs, ragged):
    return list(xs) if ragged else torch.stack(xs)


SHAPES = {"stacked_1_60x80": ([(60, 80)], False), "stacked_4_60x80": ([(60, 80)] * 4, False),
          "stacked_1_480x640": ([(480, 640)], False), "stacked_4_480x640": ([(480, 640)] * 4, False),
          "ragged": ([(60, 80), (80, 60), (61, 79)], True)}


def _prediction(torch, preds, ragged, dtype, offset, poke=True):
    """The 16-bit prediction (placed `offset` elements off), and q = p.float() placed alike."""
    p16 = [_place(torch, x, dtype, offset) for x in preds] if ragged else [_place(torch, torch.stack(preds), dtype, offset)]
    if poke:
        _poke(torch, p16[0] if ragged else p16[0][0])
    q = [_place(torch, p.float(), torch.float32, offset) for p in p16]
    return p16, q


# ------------------------------------------------------------------------------------------------
# the eager and stream-ordered calls
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(SHAPES))
@pytest.mark.parametrize("offset", [0, 1])
def test_reproj(api, torch, dtype, case, offset):
    shapes, ragged = SHAPES[case]
    T = _dt(torch, dtype)
    preds, gts, shifts, cams = _reproj_data(torch, shapes, seed=len(shapes) + offset)
    p16, q = _prediction(torch, preds, ragged, T, offset)
    s_, c = shifts.cpu().numpy(), cams.cpu().numpy()
    cam_args = (c[:, 0], s_[:, 0], s_[:, 1], CUT, SUB, c[:, 1], c[:, 2])
    g32 = [_place(torch, torch.empty_like(x), torch.float32, offset) for x in q]
    l32 = api.reproj_loss(_form(q, ragged), gts, *cam_args, outGradients=_form(g32, ragged))
    B = len(shapes)
    l32a = torch.empty(B, dtype=torch.float64, device="cuda")
    st = torch.empty(B, dtype=torch.int32, device="cuda")
    api.reproj_loss_async(_form(q, ragged), gts, shifts, cams, CUT, SUB, l32a, st)
    for s in _scales(torch, B):
        g16 = [_place(torch, torch.empty_like(x), T, offset) for x in p16]
        l16 = api.reproj_loss_amp(_form(p16, ragged), gts, *cam_args, outGradients=_form(g16, ragged), gradScale=s)
        assert l16 == l32
        _bitwise(torch, g16, _expected(torch, g32, s, T), f"eager s={s}")
        g16a = [_place(torch, torch.empty_like(x), T, offset) for x in p16]
        l16a = torch.empty(B, dtype=torch.float64, device="cuda")
        api.reproj_loss_amp_async(_form(p16, ragged), gts, shifts, cams, CUT, SUB, l16a, st, outGradients=_form(g16a, ragged),
                                  gradScale=s)
        assert torch.equal(l16a, l32a) and torch.equal(l16a.cpu(), torch.tensor(l32, dtype=torch.float64))
        assert int(st.sum()) == 0
        _bitwise(torch, g16a, _expected(torch, g32, s, T), f"async s={s}")
    # loss only
    assert api.reproj_loss_amp(_form(p16, ragged), gts, *cam_args) == l32


def _coord_shapes(case):
    shapes, ragged = SHAPES[case]
    if not ragged:
        return shapes, shapes, False
    return shapes, [(61, 80), (80, 59), (60, 80)], True   # every window one cell apart in H, W or both


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", list(SHAPES))
@pytest.mark.parametrize("offset", [0, 1])
def test_coord(api, torch, dtype, case, offset):
    pshapes, gshapes, ragged = _coord_shapes(case)
    T = _dt(torch, dtype)
    preds, gts = _coord_data(torch, pshapes, gshapes, seed=3 + offset)
    p16, q = _prediction(torch, preds, ragged, T, offset)
    gt = _stack_or_list(torch, gts, ragged)
    g32 = [_place(torch, torch.empty_like(x), torch.float32, offset) for x in q]
    l32, n32 = api.coord_loss(_form(q, ragged), gt, CUT, outGradients=_form(g32, ragged), return_counts=True)
    B = len(pshapes)
    for s in _scales(torch, B):
        g16 = [_place(torch, torch.empty_like(x), T, offset) for x in p16]
        l16, n16 = api.coord_loss_amp(_form(p16, ragged), gt, CUT, outGradients=_form(g16, ragged), return_counts=True,
                                      gradScale=s)
        assert l16 == l32 and n16 == n32
        _bitwise(torch, g16, _expected(torch, g32, s, T), f"eager s={s}")
        g16a = [_place(torch, torch.empty_like(x), T, offset) for x in p16]
        l16a = torch.empty(B, dtype=torch.float64, device="cuda")
        n16a = torch.empty(B, dtype=torch.int64, device="cuda")
        api.coord_loss_amp_async(_form(p16, ragged), gt, CUT, l16a, outGradients=_form(g16a, ragged), outCounts=n16a,
                                 gradScale=s)
        assert torch.equal(l16a.cpu(), torch.tensor(l32, dtype=torch.float64)) and n16a.tolist() == n32
        _bitwise(torch, g16a, _expected(torch, g32, s, T), f"async s={s}")
    assert api.coord_loss_amp(_form(p16, ragged), gt, CUT) == l32


@pytest.mark.parametrize("dtype", DTYPES)
def test_singular_ground_truth_zeroes_the_scaled_gradient(api, torch, dtype):
    T = _dt(torch, dtype)
    preds, gts, shifts, cams = _reproj_data(torch, [(60, 80)] * 2, seed=9)
    gts[1, :3, :3] = 0.0
    p16 = torch.stack(preds).to(T)
    g = torch.full_like(p16, 7.0)
    losses = torch.empty(2, dtype=torch.float64, device="cuda")
    status = torch.empty(2, dtype=torch.int32, device="cuda")
    api.reproj_loss_amp_async(p16, gts, shifts, cams, CUT, SUB, losses, status, outGradients=g,
                              gradScale=torch.full((1,), 3.0, device="cuda"))
    assert status.tolist() == [0, 1] and torch.isnan(losses[1]) and not torch.isnan(losses[0])
    assert torch.equal(g[1], torch.zeros_like(g[1]))


def test_grad_scale_on_the_device_is_checked(api, torch):
    p = torch.zeros(1, 3, 8, 8, dtype=torch.float16, device="cuda")
    gt = torch.ones(1, 3, 8, 8, device="cuda")
    for bad in (torch.ones(1, device="cuda", dtype=torch.float16), torch.ones(2, device="cuda")):
        with pytest.raises(RuntimeError, match="gradScale must be a CUDA float32 tensor of one element"):
            api.coord_loss_amp(p, gt, CUT, outGradients=torch.empty_like(p), gradScale=bad)


# ------------------------------------------------------------------------------------------------
# the autograd nodes
def _node_args(torch, kind, case, seed):
    """(predictions float32, call(prediction) -> loss for each of the four node entry points)."""
    import esac_b200.autograd as ag
    if kind.startswith("reproj"):
        shapes, ragged = SHAPES[case]
        preds, gts, shifts, cams = _reproj_data(torch, shapes, seed)
        s_, c = shifts.cpu().numpy(), cams.cpu().numpy()
        if kind == "reproj":
            return preds, ragged, lambda p: ag.reproj_loss(p, gts, c[:, 0], s_[:, 0], s_[:, 1], CUT, SUB, c[:, 1], c[:, 2])
        return preds, ragged, lambda p: ag.reproj_loss_async(p, gts, shifts, cams, CUT, SUB)
    pshapes, gshapes, ragged = _coord_shapes(case)
    preds, gts = _coord_data(torch, pshapes, gshapes, seed)
    gt = _stack_or_list(torch, gts, ragged)
    if kind == "coord":
        return preds, ragged, lambda p: ag.coord_loss(p, gt, CUT)
    return preds, ragged, lambda p: ag.coord_loss_async(p, gt, CUT)


def _leaves(torch, preds, ragged, dtype):
    xs = [x.to(dtype) for x in preds] if ragged else [torch.stack(preds).to(dtype)]
    _poke(torch, xs[0] if ragged else xs[0][0])
    return [x.requires_grad_() for x in xs]


def _run_node(torch, call, leaves, ragged, upcast, upstream):
    for x in leaves:
        x.grad = None
    arg = [x.float() for x in leaves] if upcast else leaves
    loss = call(_form(arg, ragged))
    (loss * upstream).backward()
    return loss.detach().clone(), [x.grad.clone() for x in leaves]


NODES = ["reproj", "coord", "reproj_async", "coord_async"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", NODES)
@pytest.mark.parametrize("case", ["stacked_4_60x80", "stacked_1_480x640", "ragged"])
def test_nodes(api, torch, dtype, kind, case):
    T = _dt(torch, dtype)
    preds, ragged, call = _node_args(torch, kind, case, seed=5)
    B = len(preds)
    api.reserve_loss_async(B, 480, 640)
    leaves = _leaves(torch, preds, ragged, T)
    for upstream in (1.0, 65536.0, 0.37):
        l16, g16 = _run_node(torch, call, leaves, ragged, False, upstream)
        l32, g32 = _run_node(torch, call, leaves, ragged, True, upstream)
        assert l16.dtype == torch.float32 and l16.shape == ()
        _bitwise(torch, l16, l32, "loss")
        _bitwise(torch, g16, g32, f"p.grad, upstream {upstream}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["reproj_async", "coord_async"])
@pytest.mark.parametrize("case", ["stacked_4_60x80", "ragged"])
def test_async_nodes_replay(api, torch, dtype, kind, case):
    """A captured forward + backward of the 16-bit stream-ordered node replays bitwise what the eager node gives, for new
    predictions and a new upstream gradient."""
    T = _dt(torch, dtype)
    preds, ragged, call = _node_args(torch, kind, case, seed=6)
    api.reserve_loss_async(len(preds), 480, 640)
    leaves = _leaves(torch, preds, ragged, T)
    upstream = torch.full((), 1024.0, device="cuda")
    _run_node(torch, call, leaves, ragged, False, upstream)   # warm-up outside the capture (first call allocates)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        for x in leaves:
            x.grad = None
        with torch.cuda.graph(graph):
            loss = call(_form(leaves, ragged))
            (loss * upstream).backward()
    torch.cuda.current_stream().wait_stream(side)
    rng = np.random.default_rng(1)
    for step in range(2):
        with torch.no_grad():
            for x in leaves:
                x.add_(torch.from_numpy(rng.standard_normal(tuple(x.shape)).astype(np.float32)).cuda().to(T) * 0.1)
            upstream.fill_(1024.0 * (step + 2))
        graph.replay()
        torch.cuda.synchronize()
        got_loss, got_grads = loss.detach().clone(), [x.grad.clone() for x in leaves]
        fresh = [x.detach().clone().requires_grad_() for x in leaves]
        want_loss, want_grads = _run_node(torch, call, fresh, ragged, False, upstream)
        _bitwise(torch, got_loss, want_loss, "replayed loss")
        _bitwise(torch, got_grads, want_grads, "replayed p.grad")


# ------------------------------------------------------------------------------------------------
# autocast training steps
def _fcn(torch, seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 16, 3, stride=2, padding=1), torch.nn.ReLU(),
                               torch.nn.Conv2d(16, 16, 3, stride=2, padding=1), torch.nn.ReLU(),
                               torch.nn.Conv2d(16, 3, 1)).cuda()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", NODES)
def test_autocast_step(api, torch, dtype, kind):
    """The p.grad that an autocast step hands the expert's 16-bit output: the 16-bit node against the p.float() route,
    with GradScaler for float16, including a scale that overflows the float16 gradient (the scaler then skips the step)."""
    T = _dt(torch, dtype)
    preds, ragged, call = _node_args(torch, kind, "stacked_4_60x80", seed=7)
    api.reserve_loss_async(4, 480, 640)
    target = torch.stack(preds)
    net = _fcn(torch, 0)
    image = torch.randn(4, 3, 240, 320, device="cuda")
    scales = [2.0 ** 16, 2.0 ** 60] if dtype == "float16" else [None]
    for init in scales:
        got = []
        for upcast in (False, True):
            scaler = torch.amp.GradScaler("cuda", init_scale=init) if init else None
            net.zero_grad()
            with torch.autocast("cuda", dtype=T):
                p = net(image)
                p.add_(target)                   # in place, as expert.py adds the scene centre: the output stays 16-bit
                assert p.dtype == T
                p.retain_grad()
                loss = call(p.float() if upcast else p)
            (scaler.scale(loss) if scaler else loss).backward()
            got.append((loss.detach().clone(), p.grad.clone()))
            if scaler:
                opt = torch.optim.SGD(net.parameters(), lr=0.0)
                scaler.step(opt)
                scaler.update()
                overflow = not bool(torch.isfinite(p.grad).all())
                assert overflow == (init > 2.0 ** 32)
                assert (scaler.get_scale() < init) == overflow
        _bitwise(torch, got[0][0], got[1][0], "loss")
        _bitwise(torch, got[0][1], got[1][1], f"p.grad, scale {init}")


def test_example_checks(torch):
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    r = subprocess.run([sys.executable, str(root / "examples" / "expert_step_autocast_synthetic.py"), "--check", "--steps", "3"],
                       capture_output=True, text=True, cwd=root, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "check passed" in r.stdout
