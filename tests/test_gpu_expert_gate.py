"""Expert gates on the H100: regions of a captured graph become conditional nodes that run where a count on the device is
positive (esac_b200.gate.ExpertGate), refused structures leave the graph as captured, the stream-ordered assignment
(api.assign_hypotheses_async) draws bitwise what the eager one draws, and the gated ESAC test and training steps match
an eager loop that runs only the experts that drew hypotheses (examples/*_gated_graph_synthetic.py)."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import esac_b200.api as api
from esac_b200.gate import ExpertGate

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu

# cudaGraphNodeType
KERNEL, CONDITIONAL = 0, 13


def _top_level_types(graph) -> list:
    """The node types of a graph's top level (the library's test hook, on the runtime the library uses)."""
    lib = api.load_library()
    n = lib.esacb200_graph_node_types(graph.raw_cuda_graph(), None, 0)
    assert n >= 0
    types = (C.c_int * max(n, 1))()
    assert lib.esacb200_graph_node_types(graph.raw_cuda_graph(), types, n) == n
    return list(types)[:n]


def _gated_adds(n, regions=None, arm=True):
    """A graph whose region i adds 1 to x[i] (and, for indices listed twice in `regions`, 10 to y[i] in a second region)."""
    regions = list(range(n)) if regions is None else regions
    x = torch.zeros(n, device="cuda")
    y = torch.zeros(n, device="cuda")
    counts = torch.zeros(n, device="cuda")
    gate = ExpertGate(n)
    seen = set()
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        if arm:
            gate.arm(counts)
        for i in regions:
            if i in seen:
                gate.run(i, lambda i=i: y[i].add_(10))
            else:
                gate.run(i, lambda i=i: x[i].add_(1))
            seen.add(i)
    return gate, graph, x, y, counts


PATTERNS = [[0, 0, 0, 0, 0, 0], [1, 1, 1, 1, 1, 1], [3, 0, 7, 0, 1, 0], [0, 2, 0, 2, 0, 2], [0.5, 0, 0, 0, 0, 0.5],
            [0, 0, 0, 0, 0, 0], [-1, float("nan"), 256, 0, 1e-30, 0]]


def test_regions_run_where_counts_are_positive():
    gate, graph, x, y, counts = _gated_adds(6)
    gate.finalize(graph)
    types = _top_level_types(graph)
    assert sorted(types) == [KERNEL] + [CONDITIONAL] * 6, types   # the arm kernel, one conditional node per region
    want = torch.zeros(6, device="cuda")
    for _ in range(2):
        for p in PATTERNS:
            counts.copy_(torch.tensor(p))
            graph.replay()
            want += (torch.tensor(p) > 0).float().cuda()
            torch.cuda.synchronize()
            assert torch.equal(x, want), (p, x, want)
    assert torch.equal(y, torch.zeros(6, device="cuda"))


def test_an_index_with_two_regions_runs_both_or_neither():
    gate, graph, x, y, counts = _gated_adds(4, regions=[0, 1, 2, 3, 1, 3])
    gate.finalize(graph)
    assert sorted(_top_level_types(graph)) == [KERNEL] + [CONDITIONAL] * 6
    for p in ([0, 1, 0, 0], [0, 0, 0, 5], [1, 1, 1, 1], [0, 0, 0, 0]):
        x0, y0 = x.clone(), y.clone()
        counts.copy_(torch.tensor(p, dtype=torch.float32))
        graph.replay()
        torch.cuda.synchronize()
        on = (torch.tensor(p) > 0).float().cuda()
        assert torch.equal(x - x0, on)
        assert torch.equal(y - y0, 10 * on * torch.tensor([0, 1, 0, 1], device="cuda"))


def _unclosed(gate, x, y):
    gate._mark(0, True)
    x[0].add_(1)
    gate.run(1, lambda: x[1].add_(1))


def _nested(gate, x, y):
    def outer():
        gate.run(1, lambda: x[1].add_(1))
        x[0].add_(1)
    gate.run(0, outer)


def _forked(gate, x, y):
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream()

    def region():
        x[0].add_(1)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            y[0].add_(1)
    gate.run(0, region)
    x[1].add_(1)
    cur.wait_stream(side)   # joins after the end marker
    y[1].add_(1)


@pytest.mark.parametrize("case, match", [(_unclosed, "has no end marker"), (_nested, "nest or overlap"),
                                         (_forked, "does not pass through its end marker"), (None, "was not armed")])
def test_refused_structures_leave_the_graph_as_captured(case, match):
    x = torch.zeros(2, device="cuda")
    y = torch.zeros(2, device="cuda")
    counts = torch.zeros(2, device="cuda")
    gate = ExpertGate(2)
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        if case is None:   # regions, but no arm
            gate.run(0, lambda: x[0].add_(1))
            gate.run(1, lambda: x[1].add_(1))
            gate.run(1, lambda: y[1].add_(1))
        else:
            gate.arm(counts)
            case(gate, x, y)
    before = _top_level_types(graph)
    with pytest.raises(RuntimeError, match=match):
        gate.finalize(graph)
    assert _top_level_types(graph) == before and CONDITIONAL not in before
    graph.replay()   # every region runs, whatever the counts say (they are 0)
    graph.replay()
    torch.cuda.synchronize()
    if case is None:
        assert x.tolist() == [2, 2] and y.tolist() == [0, 2]
    elif case is _forked:
        assert x.tolist() == [2, 2] and y.tolist() == [2, 2]
    else:
        assert x.tolist() == [2, 2]


def test_finalize_twice_and_without_keep_graph():
    gate, graph, x, y, counts = _gated_adds(3)
    gate.finalize(graph)
    with pytest.raises(RuntimeError, match="no region of this gate"):
        gate.finalize(graph)
    counts.copy_(torch.tensor([0.0, 1.0, 0.0]))
    graph.replay()
    torch.cuda.synchronize()
    assert x.tolist() == [0, 1, 0]
    plain = torch.cuda.CUDAGraph()
    g2 = ExpertGate(1)
    with torch.cuda.graph(plain):
        g2.arm(counts[:1])
        g2.run(0, lambda: x[0].add_(1))
    with pytest.raises(RuntimeError, match="keep_graph=True"):
        g2.finalize(plain)


def test_arm_and_mark_need_a_capture():
    gate = ExpertGate(2)
    with pytest.raises(RuntimeError, match="works only while the stream is being captured"):
        gate._ctx.check(gate._ctx.lib.esacb200_gate_arm(gate._handle, torch.zeros(2, device="cuda").data_ptr(),
                                                        torch.cuda.current_stream().cuda_stream))
    with pytest.raises(RuntimeError, match="works only while the stream is being captured"):
        gate._mark(0, True)
    with pytest.raises(RuntimeError, match=r"index 2 outside \[0, 2\)"):
        gate._mark(2, True)


# ---- the stream-ordered assignment -------------------------------------------------------------------------------------
MODES = [dict(), dict(maxExperts=2), dict(expertSelection=True), dict(maxExperts=3, expertSelection=True)]


def _probs(B, E, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(3 * torch.randn(B, E, generator=g), dim=1).cuda()


def _async_draw(probs, M, seed_t, **mode):
    lead = tuple(probs.shape[:-1])
    a = torch.empty(lead + (M,), dtype=torch.int64, device="cuda")
    h = torch.empty(lead + (probs.shape[-1],), device="cuda")
    s = torch.full(lead, -7, dtype=torch.int32, device="cuda")
    api.assign_hypotheses_async(probs, M, seed_t, a, h, s, **mode)
    return a, h, s


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("mode", range(len(MODES)))
def test_assign_async_is_the_eager_draw(B, mode):
    kw = MODES[mode]
    probs = _probs(B, 6, 10 * B + mode)
    for seed in (0, 2020, (1 << 63) - 5):
        a_ref, h_ref = api.assign_hypotheses(probs, 256, seed, **kw)
        a, h, s = _async_draw(probs, 256, torch.tensor([seed], dtype=torch.int64, device="cuda"), **kw)
        torch.cuda.synchronize()
        assert torch.equal(a, a_ref) and torch.equal(h, h_ref) and s.tolist() == [0] * B
    if B == 1:   # one image as [E] / [M] / [] tensors
        a, h, s = _async_draw(probs[0], 256, torch.tensor(2020, dtype=torch.int64, device="cuda"), **kw)
        a_ref, h_ref = api.assign_hypotheses(probs, 256, 2020, **kw)
        assert torch.equal(a, a_ref[0]) and torch.equal(h, h_ref[0]) and int(s) == 0


def test_assign_async_in_a_graph_advances_its_seed():
    probs = _probs(4, 6, 5)
    seed = torch.tensor([123], dtype=torch.int64, device="cuda")
    a = torch.empty(4, 64, dtype=torch.int64, device="cuda")
    h = torch.empty(4, 6, device="cuda")
    s = torch.empty(4, dtype=torch.int32, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        api.assign_hypotheses_async(probs, 64, seed, a, h, s, maxExperts=2)
        seed.add_(1)
    for j in range(4):
        graph.replay()
        a_ref, h_ref = api.assign_hypotheses(probs, 64, 123 + j, maxExperts=2)
        assert torch.equal(a, a_ref) and torch.equal(h, h_ref) and s.tolist() == [0] * 4
    seed.fill_(9)   # or the caller writes the next seed before a replay
    graph.replay()
    assert torch.equal(a, api.assign_hypotheses(probs, 64, 9, maxExperts=2)[0])


def test_assign_async_reports_a_bad_distribution_in_its_status():
    probs = _probs(4, 5, 1)
    probs[1, 2] = -0.5
    probs[2] = 0
    probs[3, 0] = float("inf")
    a, h, s = _async_draw(probs, 32, torch.tensor([1], dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    assert s.tolist() == [0, 1, 2, 1]
    assert torch.equal(a[0], api.assign_hypotheses(probs[:1], 32, 1)[0][0])
    for bad in (1, 2, 3):
        with pytest.raises(RuntimeError):
            api.assign_hypotheses(probs[bad:bad + 1], 32, 1)


# ---- the gated ESAC steps -----------------------------------------------------------------------------------------------
def _example(name):
    import importlib.util
    sys.path.insert(0, str(ROOT / "examples"))
    spec = importlib.util.spec_from_file_location(name, ROOT / "examples" / f"{name}.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture
def cudnn_fixed():
    """The examples fix cuDNN's algorithm choice so that eager and captured convolutions agree bitwise; restored after.
    They also run on a context of their own, whose stream-ordered workspace no earlier capture has frozen."""
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    saved = api._contexts.get(0)
    api._contexts[0] = api.Context(0)
    yield
    torch.cuda.synchronize()
    if saved is not None:
        api._contexts[0] = saved
    else:
        api._contexts.pop(0, None)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


def test_gated_test_step_is_the_eager_loop_over_active_experts(cudnn_fixed, capsys):
    """E = 6, maxExperts = 2: at least 4 experts idle on every image; 8 replays bitwise the eager loop."""
    rc = _example("test_step_gated_graph_synthetic").main(["--images", "8", "--experts", "6", "--maxexperts", "2", "--check"])
    out = capsys.readouterr().out
    assert rc == 0, out
    runs = [line for line in out.splitlines() if line.startswith("image ")]
    assert len(runs) == 8 and all("bitwise equal" in line for line in runs), out
    for line in runs:
        active = eval(line.split("experts run ")[1].split("]")[0] + "]")
        assert 1 <= len(active) <= 2, line


def test_gated_train_step_is_the_eager_loop_over_active_experts(cudnn_fixed, capsys):
    """5 replays: loss, coordinate gradient, every parameter and Adam state bitwise the eager twin's; idle experts
    untouched."""
    rc = _example("train_step_gated_graph_synthetic").main(["--images", "5", "--experts", "6", "--maxexperts", "2",
                                                            "--check"])
    out = capsys.readouterr().out
    assert rc == 0, out
    runs = [line for line in out.splitlines() if line.startswith("image ")]
    assert len(runs) == 5, out
    assert all("idle experts untouched" in line and "eager loop: bitwise equal" in line for line in runs), out


def test_the_ungated_graph_moves_an_idle_expert(cudnn_fixed):
    """The control: the same step with every region run (examples/train_step_graph_synthetic.py's behaviour) moves an
    expert that drew no hypotheses."""
    ex = _example("train_step_gated_graph_synthetic")
    from test_step_graph_synthetic import PerImageFocalDataset
    opt = ex.parse(["--images", "1", "--experts", "6", "--maxexperts", "2"])
    trainset = PerImageFocalDataset(num_experts=6, length=1, hypotheses=opt.hypotheses, seed=3)
    T = ex.GatedTraining(opt, trainset, ex.AlwaysGate())
    graph, loss, grad = T.capture()
    T.load(trainset, 0)
    before = [[t.clone() for t in ex.tensors_of(m, o)] for m, o in zip(T.experts, T.opts)]
    graph.replay()
    torch.cuda.synchronize()
    idle = [e for e in range(6) if float(T.hist[e]) == 0]
    assert len(idle) >= 4
    for e in idle:
        after = ex.tensors_of(T.experts[e], T.opts[e])
        assert not ex.same(before[e], after)
        assert float(after[len(list(T.experts[e].parameters()))]) == float(before[e][len(list(T.experts[e].parameters()))]) + 1


@pytest.mark.parametrize("name", ["test_step_gated_graph_synthetic", "train_step_gated_graph_synthetic"])
def test_gated_examples_check(name):
    r = subprocess.run([sys.executable, str(ROOT / "examples" / f"{name}.py"), "--check"], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
