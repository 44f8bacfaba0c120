"""The sharded forward and backward on one GPU, held to the unsharded calls (run with `-m gpu`).

A sharded call runs one shard of the experts or of the hypotheses, and the ranks merge their shards in one all-gather
(forward) or two small exchanges (backward: the softmax normalisation, then the expected loss).  Every call here is
deterministic under option fixed_seed with the same seed, so the shards can run one after another on one context:
  * backward over the exchange callback, by replay.  Pass A records each shard's (max, sum exp) pair, pass B answers with
    the merged pair and records the shard's partial expectation, pass C answers both exchanges with the merged values;
  * forward records: each shard's esacb200_forward_pack record, field by field, then the records stitched and selected;
  * the library's NCCL communicator with one rank: every collective, and every kernel around it, runs;
  * the two merge kernels (select_gathered_kernel, rescale_probs_gathered_kernel) through esacb200_test_gathered, on records
    and pairs built here, against sharded.select_global and float64 numpy.
Collectives between two devices are tests/test_gpu_multi.py's (it needs two GPUs).

Bars: bitwise where the merge is the identity (one shard, one rank).  Over 2 and more shards the probabilities differ from
the unsharded ones by the rounding of the merged normalisation, and the refined poses by the refinement group, which follows
the shard's count of contributing hypotheses.  The bars below are about 10x the worst difference measured on an H100 SXM
(80 GB, 700 W) over every layout of this file."""
import math

import numpy as np
import pytest

import grad_terms as GT
from esac_b200.synth import make_scene
from oracle import esac_oracle as O
from ref_golden_util import GOLD_DIR, load, params_of
from test_gpu_backward import BAR_SCENES
from test_gpu_ref_golden import BAR_SAMPLED, BAR_SMALL
from esac_b200 import sharded

pytestmark = pytest.mark.gpu

SEED = 5
ARGS = (1.0, 100.0, 100.0)      # wLossRot, wLossTrans, lossCut
# measured worst over the layouts: 2 ulp; 1.2e-15 (expected loss), 1.9e-17 (per-hypothesis losses); expert-major gradients
# bitwise the unsharded ones; hypothesis-major 1.2e-7 of a class's largest entry, the float32 rounding of the sum over the shards
PROB_ULPS = 20                  # probabilities of 2+ shards against the unsharded ones, in ulp of the unsharded value
LOSS_BAR = 1.2e-14              # expected loss and per-hypothesis losses of 2+ shards, relative to max(1, |unsharded|)
GRAD_BAR = 1e-12                # expert-major gradient of 2+ shards, class by class against the unsharded one
GRAD_BAR_SUMMED = 1.2e-6        # hypothesis-major: the shards' float32 gradients summed on the host
NEUTRAL = (-1e300, 0.0)         # what a shard without hypotheses contributes to exchange 1 (sharded.backward_sharded)


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def api():
    """The module's own context with fixed_seed; the shared one is restored afterwards."""
    import esac_b200.api as api
    saved = api._contexts.get(0)
    ctx = api.Context(0)
    api._contexts[0] = ctx
    ctx.set_option("fixed_seed", 1)
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


# ---- scenes and layouts -------------------------------------------------------------------------------------------------------
def _scene(name):
    if name == "even":        # 5 experts of 24 hypotheses each, contiguous per expert
        return make_scene(E=5, H=30, W=40, M=24, sub=8, seed=77, per_expert=True, active_only=False)
    if name == "peaked":      # 90 % of the hypotheses on the ground-truth expert (3), sorted so that experts are contiguous
        sc = make_scene(E=5, H=60, W=80, M=120, sub=8, seed=3, gt_mass=0.9, active_only=False)
        sc.assign = np.sort(sc.assign)
        return sc
    if name == "full":        # 480x640 maps: the TMA scoring path and the refinement groups of a full-size map
        return make_scene(E=4, H=480, W=640, M=16, sub=1, seed=21, per_expert=True, active_only=False)
    raise KeyError(name)


class Shard:
    """One rank's inputs: planes [e0, e1) of `coords` (hypothesis-major: all of them) and the global hypotheses gidx, which are
    hyp_offset + k * hyp_stride unless `injected` (the minimal sets are then given, and the dealing does not matter)."""

    def __init__(self, coords, assign, e0, e1, gidx, hyp_offset, hyp_stride, torch, injected=False):
        self.e0, self.e1, self.gidx = e0, e1, np.asarray(gidx, np.int64)
        self.hyp_offset, self.hyp_stride, self.M = int(hyp_offset), int(hyp_stride), len(gidx)
        assert injected or np.array_equal(self.gidx, self.hyp_offset + self.hyp_stride * np.arange(self.M))
        planes = coords[e0:e1] if e1 > e0 else np.zeros((1,) + coords.shape[1:], np.float32)
        self.coords = torch.from_numpy(np.ascontiguousarray(planes)).cuda()
        self.assign = torch.from_numpy(np.ascontiguousarray(assign[self.gidx] - e0)).cuda()


def _expert_major(coords, assign, sizes, torch, injected=False):
    shards, e0 = [], 0
    for n in sizes:
        gidx = np.flatnonzero((assign >= e0) & (assign < e0 + n))
        shards.append(Shard(coords, assign, e0, e0 + n, gidx, gidx[0] if gidx.size else 0, 1, torch, injected))
        e0 += n
    assert e0 == coords.shape[0]
    return shards


def _hypothesis_major(sc, world, strided, torch):
    M, E = len(sc.assign), sc.coords.shape[0]
    if strided:
        return [Shard(sc.coords, sc.assign, 0, E, np.arange(r, M, world), r, world, torch) for r in range(world)]
    cuts = [round(M * r / world) for r in range(world + 1)]
    return [Shard(sc.coords, sc.assign, 0, E, np.arange(cuts[r], cuts[r + 1]), cuts[r], 1, torch) for r in range(world)]


# (scene, kind, argument): expert-major shard sizes, or the world of a hypothesis-major layout
LAYOUTS = {
    "world1": ("even", "experts", [5]),
    "world2": ("even", "experts", [3, 2]),
    "world3": ("even", "experts", [2, 2, 1]),
    "world5": ("even", "experts", [1, 1, 1, 1, 1]),
    "empty_shard": ("even", "experts", [2, 0, 3]),
    "peaked": ("peaked", "experts", [3, 2]),
    "hyp_contiguous": ("even", "contiguous", 2),
    "hyp_strided": ("even", "strided", 3),
    "full_world2": ("full", "experts", [2, 2]),
    "full_strided": ("full", "strided", 2),
}
BACKWARD_LAYOUTS = list(LAYOUTS)
FORWARD_LAYOUTS = BACKWARD_LAYOUTS + ["hyp_stride2"]
LAYOUTS["hyp_stride2"] = ("even", "strided", 2)


def _layout(name, sc, torch):
    _, kind, arg = LAYOUTS[name]
    return _expert_major(sc.coords, sc.assign, arg, torch) if kind == "experts" else _hypothesis_major(sc, arg, kind == "strided", torch)


_CACHE = {}


def _reference(api, torch, name, oracle=True):
    """The scene, and the unsharded backward and forward on it (and the cv2 oracle's backward with its gradient classes)."""
    if name in _CACHE and (not oracle or "g_oracle" in _CACHE[name]):
        return _CACHE[name]
    sc = _scene(name)
    ref = _CACHE.get(name) or {"sc": sc}
    if "loss" not in ref:
        ctx = api.context(0)
        coords, assign = torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda()
        g = torch.zeros_like(coords)
        api.set_seed(SEED)
        ref["loss"] = api.backward(coords, g, assign, torch.from_numpy(sc.gt_pose), *ARGS, *sc.params)
        ref["g"] = g.cpu().numpy()
        ref["hyp"] = ctx.hypotheses(losses=True)
        ref["n_contrib"] = ctx.stats()["n_contrib"]
        out = np.zeros((4, 4), np.float32)
        api.set_seed(SEED)
        ref["expert"] = api.forward(coords, assign, out, *sc.params)
        ref["pose"] = out
        ref["winner"] = ctx.stats()["winner"]
        ref["fwd_scores"] = ctx.hypotheses()["scores"]
    if oracle:
        g_ref = np.zeros_like(sc.coords)
        l_ref, bt = O.backward(sc.coords, g_ref, sc.assign, sc.gt_pose, *ARGS, *sc.params, seed=SEED, trace=True)
        ref.update(l_oracle=l_ref, g_oracle=g_ref, classes=GT.cell_classes(sc.coords.shape, sc.assign, bt))
    _CACHE[name] = ref
    return ref


# ---- (a) backward over the exchange callback, by replay -------------------------------------------------------------------------
def _backward_shard(api, torch, shard, gt, loss_args, params, replies, cells=None):
    """One esacb200_backward_sharded call on `shard`; the callback answers phase p with replies[p] (default: the values it was
    given) and records every call.  Returns the loss, a fresh gradient and the calls."""
    calls = []

    def exchange(phase, values):
        calls.append((phase, list(values)))
        return list(replies.get(phase, values))

    ctx = api.context(0)
    g = torch.zeros_like(shard.coords)
    ctx.set_option("hyp_stride", shard.hyp_stride)
    try:
        if cells is not None:
            ctx.inject_cells(cells)
        api.set_seed(SEED)
        loss = api.backward_sharded(shard.coords, g, shard.assign, gt, *loss_args, *params, exchange=exchange,
                                    hyp_offset=shard.hyp_offset)
    finally:
        ctx.set_option("hyp_stride", 1)
    assert [(p, len(v)) for p, v in calls] == [(1, 2), (2, 1)], calls
    return loss, g.cpu().numpy(), calls


def replay_backward(api, torch, shards, gt, params, loss_args=ARGS, cells_of=None):
    """Passes A, B and C over every shard; returns the global loss, each shard's gradient, hypotheses and statistics."""
    ctx = api.context(0)
    cells = (lambda s: None) if cells_of is None else cells_of
    pairs = []
    for s in shards:                                   # pass A: the shard's own (max, sum exp)
        pairs.append(NEUTRAL if s.M == 0 else tuple(_backward_shard(api, torch, s, gt, loss_args, params, {}, cells(s))[2][0][1]))
    gmax = max(m for m, _ in pairs)                    # merged as sharded.make_exchange and rescale_probs_gathered_kernel do
    gsum = 0.0
    for m, v in pairs:
        gsum += v * math.exp(m - gmax)
    partials = []
    for s, pair in zip(shards, pairs):                 # pass B: the merged pair in, the partial expectation out
        if s.M == 0:
            partials.append(0.0)
            continue
        calls = _backward_shard(api, torch, s, gt, loss_args, params, {1: [gmax, gsum]}, cells(s))[2]
        assert tuple(calls[0][1]) == pair
        partials.append(calls[1][1][0])
    total = 0.0
    for p in partials:
        total += p
    out = []
    for s, pair, part in zip(shards, pairs, partials):  # pass C: both merged values in; its gradient is the result
        if s.M == 0:
            out.append(None)
            continue
        loss, g, calls = _backward_shard(api, torch, s, gt, loss_args, params, {1: [gmax, gsum], 2: [total]}, cells(s))
        assert tuple(calls[0][1]) == pair and calls[1][1] == [part]      # bitwise pass A's and pass B's inputs
        assert loss == total
        out.append({"g": g, "hyp": ctx.hypotheses(losses=True), "stats": ctx.stats()})
    return total, out


def _assemble(sc, shards, res):
    """The shards' gradients placed in (expert-major) or summed over (hypothesis-major) the full tensor, and their hypotheses
    in global order."""
    M = len(sc.assign)
    g = np.zeros(sc.coords.shape, np.float64)
    hyp = {k: np.full(M, np.nan) for k in ("probs", "losses", "scores")}
    for s, r in zip(shards, res):
        if r is None:
            continue
        g[s.e0:s.e1] += r["g"]
        for k in hyp:
            hyp[k][s.gidx] = r["hyp"][k]
    return g, hyp


def _measure(name, what, value):
    print(f"MEASURED {name} {what} {value:.3e}")
    return value


@pytest.mark.parametrize("name", BACKWARD_LAYOUTS)
def test_backward_by_replay_matches_the_unsharded_call(api, torch, name):
    scene = LAYOUTS[name][0]
    ref = _reference(api, torch, scene, oracle=scene != "full")
    sc = ref["sc"]
    shards = _layout(name, sc, torch)
    assert sorted(np.concatenate([s.gidx for s in shards]).tolist()) == list(range(len(sc.assign)))
    loss, res = replay_backward(api, torch, shards, torch.from_numpy(sc.gt_pose), sc.params)
    g, hyp = _assemble(sc, shards, res)
    if len(shards) == 1:       # the merge is the identity: bitwise esac.backward
        assert loss == ref["loss"]
        assert np.array_equal(res[0]["g"], ref["g"])
        assert np.array_equal(hyp["probs"], ref["hyp"]["probs"])
        return
    p_ref = ref["hyp"]["probs"]
    contrib = hyp["probs"] >= O.PROB_THRESH
    assert np.array_equal(contrib, p_ref >= O.PROB_THRESH)
    assert sum(r["stats"]["n_contrib"] for r in res if r is not None) == ref["n_contrib"]
    assert abs(hyp["probs"].sum() - 1.0) < 1e-12
    ulps = _measure(name, "probs_ulp", float((np.abs(hyp["probs"] - p_ref) / np.spacing(np.maximum(p_ref, 1e-300))).max()))
    assert ulps <= PROB_ULPS
    assert np.array_equal(hyp["scores"], ref["hyp"]["scores"])
    lscale = max(1.0, np.abs(ref["hyp"]["losses"]).max())
    dl = _measure(name, "hyp_losses", float(np.abs(hyp["losses"] - ref["hyp"]["losses"]).max() / lscale))
    assert dl <= LOSS_BAR
    dL = _measure(name, "loss", abs(loss - ref["loss"]) / max(1.0, abs(ref["loss"])))
    assert dL <= LOSS_BAR
    summed = LAYOUTS[name][1] != "experts"
    if "classes" in ref:
        rep = GT.compare(g, ref["g"], ref["classes"])
        worst = _measure(name, "grad_vs_unsharded", max(rep[n]["rel"] for n in GT.NAMES))
        assert worst <= (GRAD_BAR_SUMMED if summed else GRAD_BAR), GT.fmt(rep)
        rep = GT.assert_classwise(g, ref["g_oracle"], ref["classes"], BAR_SCENES, f"{name} against the oracle")
        print(f"{name} against the oracle: {GT.fmt(rep)}")
    else:                       # 480x640: no oracle; against the unsharded gradient relative to its largest entry
        rel = _measure(name, "grad_vs_unsharded", float(np.abs(g - ref["g"]).max() / np.abs(ref["g"]).max()))
        assert rel <= (GRAD_BAR_SUMMED if summed else GRAD_BAR)
    if name == "peaked":
        # the shard of the outlier experts holds hypotheses, several of which its own softmax keeps, but the global one none
        s0, r0 = shards[0], res[0]
        assert s0.M >= 2 and r0["stats"]["n_contrib"] == 0
        own = np.exp(r0["hyp"]["scores"] - r0["hyp"]["scores"].max())
        assert ((own / own.sum()) >= O.PROB_THRESH).sum() >= 2
        assert not contrib[s0.gidx].any()


@pytest.mark.parametrize("fixture,sizes", [("ref_ensemble3_30x40_shift", [2, 1]), ("ref_full_7x480x640", [4, 3])])
def test_backward_by_replay_matches_the_compiled_reference(api, torch, fixture, sizes):
    """Expert-major shards of a compiled-reference fixture, each with its slice of the fixture's minimal sets injected."""
    z, coords = load(GOLD_DIR / f"{fixture}.npz")
    params = params_of(z)
    cells, assign = z["cells"], z["assign"]
    shards = _expert_major(coords, assign, sizes, torch, injected=True)
    w_rot, w_trans, cut = (float(v) for v in z["loss_args"])
    loss, res = replay_backward(api, torch, shards, torch.from_numpy(z["gt_pose"]), params, (w_rot, w_trans, cut),
                                cells_of=lambda s: np.ascontiguousarray(cells[s.gidx]))
    g = np.zeros(coords.shape, np.float32)
    for s, r in zip(shards, res):
        g[s.e0:s.e1] = r["g"]
    assert abs(loss - float(z["loss"])) < 1e-6 * max(1.0, abs(float(z["loss"])))
    if "grads" in z.files:
        scale = max(np.abs(z["grads"]).max(), 1e-12)
        assert np.abs(g - z["grads"]).max() / scale < 1e-3
        _, bt = O.backward(coords, np.zeros_like(coords), assign, z["gt_pose"], w_rot, w_trans, cut, *params,
                           injected_cells=cells, trace=True)
        rep = GT.assert_classwise(g, z["grads"], GT.cell_classes(coords.shape, assign, bt), BAR_SMALL, fixture)
        print(f"{fixture} sharded {sizes}: {GT.fmt(rep)}")
    else:
        scale = float(z["grad_max"])
        got = g.reshape(-1)[z["grad_idx"]].astype(np.float64)
        assert np.abs(got - z["grad_val"]).max() / scale < 1e-3
        other = ~GT.sampled_classes(z["grad_idx"], g.shape, assign, cells[:, -1], O.softmax(z["oracle_scores"]))
        oscale = max(np.abs(z["grad_val"][other]).max(), GT.FLOOR * scale)
        rel = np.abs(got[other] - z["grad_val"][other]).max() / oscale
        print(f"{fixture} sharded {sizes}: other {rel:.2e} of {oscale:.2e}")
        assert rel <= BAR_SAMPLED
        pa = np.abs(g).astype(np.float64).sum(axis=(2, 3))
        assert np.abs(g.astype(np.float64).sum(axis=(2, 3)) - z["grad_plane_sum"]).max() < 1e-3 * z["grad_plane_abs"].max()
        assert np.abs(pa - z["grad_plane_abs"]).max() < 1e-3 * z["grad_plane_abs"].max()


# ---- (b) forward records ------------------------------------------------------------------------------------------------------
def _pack(api, torch, shard, params, M_pad, expert_offset):
    ctx = api.context(0)
    buf = torch.full((M_pad + api.PACK_TAIL,), 7.0, dtype=torch.float64, device="cuda")
    ctx.set_option("hyp_offset", shard.hyp_offset)
    ctx.set_option("hyp_stride", shard.hyp_stride)
    try:
        api.set_seed(SEED)
        api.forward_pack(shard.coords, shard.assign, params, expert_offset, buf, M_pad=M_pad)
        rec = buf.cpu().numpy()
        own = None
        if shard.M > 0:        # the shard alone through esac.forward: its winner, pose and (local) expert
            out = np.zeros((4, 4), np.float32)
            api.set_seed(SEED)
            e = api.forward(shard.coords, shard.assign, out, *params)
            own = (e, out, ctx.stats()["winner"])
    finally:
        ctx.set_option("hyp_offset", 0)
        ctx.set_option("hyp_stride", 1)
    return rec, own


def _select_ref(gathered, M_pad):
    """float64 restatement of draw(training = false) over records: the largest score, ties to the lowest global index; returns
    (rank, global index) or None when no record holds a hypothesis."""
    best = None
    for r, rec in enumerate(gathered):
        t = rec[M_pad:]
        for k in range(int(t[18])):
            key = (-rec[k], int(t[19]) + k * int(t[20]))
            if best is None or key < best[0]:
                best = (key, r)
    return None if best is None else (best[1], best[0][1])


def _select_on_device(api, torch, gathered, M_pad):
    """esacb200_test_gathered's selection: the 20 floats of the ForwardRecord."""
    ctx = api.context(0)
    g = torch.from_numpy(np.ascontiguousarray(gathered, np.float64)).cuda()
    out = torch.zeros(20, dtype=torch.float32, device="cuda")
    ctx.check(ctx.lib.esacb200_test_gathered(ctx.handle, g.shape[0], M_pad, g.data_ptr(), out.data_ptr(), None, None, 0, None,
                                             None, None, None))
    o = out.cpu().numpy()
    return {"pose": o[:16].reshape(4, 4), "expert": o[16], "bad": o[17], "winner": o[18], "rank": o[19]}


@pytest.mark.parametrize("name", FORWARD_LAYOUTS)
def test_forward_records_match_the_unsharded_forward(api, torch, name):
    ref = _reference(api, torch, LAYOUTS[name][0], oracle=False)
    sc = ref["sc"]
    shards = _layout(name, sc, torch)
    M_pad = max(max(s.M for s in shards), 1)
    recs = []
    for s in shards:
        rec, own = _pack(api, torch, s, sc.params, M_pad, s.e0)
        t = rec[M_pad:]
        assert np.array_equal(rec[:s.M], ref["fwd_scores"][s.gidx])          # bitwise the unsharded forward's scores
        assert np.all(rec[s.M:M_pad] == -np.inf)
        assert (t[18], t[19], t[20]) == (s.M, s.hyp_offset, s.hyp_stride)
        if s.M == 0:
            assert np.all(t[:18] == -1.0)
        else:
            e, pose, winner = own
            assert t[16] == s.e0 + e                                          # the global expert
            assert t[17] == winner == int(np.argmax(rec[:s.M]))               # the local winner: first maximum
            assert np.array_equal(t[:16].astype(np.float32).reshape(4, 4), pose)
            assert np.array_equal(t[:16], t[:16].astype(np.float32))
        recs.append(rec)
    gathered = np.stack(recs)
    w, rank, pose, expert, probs = sharded.select_global(gathered, M_pad)
    assert expert == ref["expert"]
    assert np.array_equal(pose, ref["pose"])          # the winner is refined on the same plane with the same group
    dev = _select_on_device(api, torch, gathered, M_pad)
    assert (dev["expert"], dev["bad"], dev["winner"], dev["rank"]) == (ref["expert"], 0, ref["winner"], rank)
    assert np.array_equal(dev["pose"], ref["pose"])


def test_forward_record_of_a_bad_shard_names_no_expert(api, torch):
    """A shard whose hypAssignment holds an index outside its planes writes expert -1, and the selection flags it."""
    sc = _scene("even")
    s = _expert_major(sc.coords, sc.assign, [3, 2], torch)[1]
    s.assign[5] = 2                             # the shard has planes 0 and 1
    buf = torch.zeros(s.M + api.PACK_TAIL, dtype=torch.float64, device="cuda")
    api.set_seed(SEED)
    api.forward_pack(s.coords, s.assign, sc.params, s.e0, buf, M_pad=s.M)
    rec = buf.cpu().numpy()
    assert rec[s.M + 16] == -1.0 and rec[s.M + 18] == s.M
    assert _select_on_device(api, torch, rec[None], s.M)["bad"] == 1.0


# ---- (c) the library's communicator with one rank -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def one_rank(api):
    ctx = api.context(0)
    try:
        uid = api.nccl_unique_id()
    except RuntimeError as e:
        pytest.skip(f"libnccl.so.2 cannot be loaded: {e}")
    ctx.comm_init(1, 0, uid)
    try:
        yield ctx
    finally:
        ctx.comm_destroy()


@pytest.mark.parametrize("repeat", [0, 1])
def test_one_rank_communicator_is_bitwise_the_unsharded_calls(api, torch, one_rank, repeat):
    """Every collective of the NCCL entry points with world 1: bitwise esac.forward / esac.backward.  Run twice on the same
    context, so that a work buffer left holding the previous call's values shows."""
    print(f"one-rank NCCL communicator initialised on {torch.cuda.get_device_name(0)}")
    ref = _reference(api, torch, "even", oracle=False)
    sc = ref["sc"]
    coords, assign = torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda()
    gt = torch.from_numpy(sc.gt_pose)
    for c, a, out in ((coords, assign, torch.zeros(4, 4, device="cuda")),
                      (coords.cpu(), assign.cpu(), torch.zeros(4, 4))):
        api.set_seed(SEED)
        e = api.forward_sharded(c, a, out, *sc.params, expert_offset=0, M_pad=len(sc.assign), device=0)
        assert e == ref["expert"] and np.array_equal(out.cpu().numpy(), ref["pose"])
    g = torch.zeros_like(coords)
    api.set_seed(SEED)
    loss = api.backward_sharded_nccl(coords, g, assign, gt, *ARGS, *sc.params)
    assert loss == ref["loss"] and np.array_equal(g.cpu().numpy(), ref["g"])
    # hypothesis-major: the reduced gradient is added to the caller's tensor
    g = torch.full_like(coords, 0.5)
    api.set_seed(SEED)
    loss = api.backward_sharded_nccl(coords, g, assign, gt, *ARGS, *sc.params, reduce_grads=True)
    assert loss == ref["loss"]
    assert np.array_equal(g.cpu().numpy(), (np.float32(0.5) + ref["g"]).astype(np.float32))
    # a rank without hypotheses: loss 0, gradient untouched
    empty = torch.zeros(0, dtype=torch.int64, device="cuda")
    for reduce in (False, True):
        g = torch.full_like(coords, 0.5)
        api.set_seed(SEED)
        loss = api.backward_sharded_nccl(coords, g, empty, gt, *ARGS, *sc.params, reduce_grads=reduce)
        assert loss == 0.0 and bool((g == 0.5).all())
    # ... and a forward in which no rank holds a hypothesis is refused
    with pytest.raises(RuntimeError, match="no shard holds a hypothesis"):
        api.forward_sharded(coords, empty, torch.zeros(4, 4, device="cuda"), *sc.params, expert_offset=0, M_pad=1)


# ---- the merge kernels through esacb200_test_gathered ------------------------------------------------------------------------
def _records(rng, world, M_pad, Ms, strided, levels=6):
    """Records with scores on a coarse grid (exact ties, no near ties), -inf padding, contiguous or strided dealing."""
    total = sum(Ms)
    g = np.full((world, M_pad + 21), -np.inf)
    off = 0
    for r in range(world):
        M = Ms[r]
        g[r, :M] = rng.integers(0, levels, M) * 0.5
        t = g[r, M_pad:]
        t[:16] = rng.integers(-100, 100, 16) * 0.25 if M else -1.0
        t[16], t[17] = (rng.integers(0, 50), rng.integers(0, max(M, 1))) if M else (-1.0, -1.0)
        t[18] = M
        if strided:      # hypothesis h to rank h % world (every rank's M is then ceil((total - r) / world))
            t[19], t[20] = r, world
        else:
            t[19], t[20] = off, 1
        off += M
    return g, total


def _check_select(api, torch, g, M_pad):
    dev = _select_on_device(api, torch, g, M_pad)
    want = _select_ref(g, M_pad)
    if want is None:
        assert (dev["winner"], dev["rank"], dev["expert"]) == (-1, -1, -1)
        return dev
    rank, gi = want
    assert (dev["rank"], dev["winner"]) == (rank, gi)
    assert dev["expert"] == g[rank, M_pad + 16]
    assert np.array_equal(dev["pose"], g[rank, M_pad:M_pad + 16].astype(np.float32).reshape(4, 4))
    _, r2, pose, expert, _ = sharded.select_global(g, M_pad)      # the host selection of the torch.distributed transport
    assert (r2, expert) == (rank, g[rank, M_pad + 16]) and np.array_equal(pose, dev["pose"])
    return dev


@pytest.mark.parametrize("M_pad", [1, 255, 256, 257, 4096])
@pytest.mark.parametrize("world", [1, 2, 3, 8, 64])
@pytest.mark.parametrize("strided", [False, True], ids=["contiguous", "strided"])
def test_select_gathered_matches_the_host_selection(api, torch, world, M_pad, strided):
    rng = np.random.default_rng(world * 10007 + M_pad * 3 + strided)
    if strided:
        total = world * M_pad - int(rng.integers(0, world))
        Ms = [len(range(r, total, world)) for r in range(world)]
    else:
        Ms = [int(rng.integers(0, M_pad + 1)) for _ in range(world)]
        Ms[-1] = max(Ms[-1], 1)
    g, _ = _records(rng, world, M_pad, Ms, strided)
    dev = _check_select(api, torch, g, M_pad)
    assert dev["bad"] == 0
    # equal maxima in the same rank, in different ranks and in different warps of the block: the unsharded order wins
    top = g[:, :M_pad].max() + 1.0
    slots = [(r, k) for r in range(world) for k in range(Ms[r])]
    picks = [slots[i] for i in rng.choice(len(slots), size=min(len(slots), 5), replace=False)]
    picks += [slots[-1], slots[0]] + ([(world - 1, 0)] if Ms[-1] else [])
    for r, k in picks:
        g[r, k] = top
    _check_select(api, torch, g, M_pad)
    if strided and world > 1:     # rank 1's slot 0 is hypothesis 1, before rank 0's slot 1 (hypothesis world)
        g2 = g.copy()
        g2[:, :M_pad] = np.where(np.isfinite(g2[:, :M_pad]), 0.0, -np.inf)
        if Ms[0] > 1 and Ms[1] > 0:
            g2[0, 1] = g2[1, 0] = 1.0
            assert _check_select(api, torch, g2, M_pad)["rank"] == 1
    if world > 1:                 # an empty shard at rank 0
        g[0, :M_pad], g[0, M_pad:M_pad + 18], g[0, M_pad + 18] = -np.inf, -1.0, 0
        _check_select(api, torch, g, M_pad)


def test_select_gathered_edges(api, torch):
    rng = np.random.default_rng(3)
    # equal maxima in different warps of one rank, at slots 31 / 32 and 255 / 256 of the block-stride loop
    for a, b in ((31, 32), (255, 256), (3, 4000), (4000, 3)):
        g, _ = _records(rng, 1, 4096, [4096], False)
        g[0, a] = g[0, b] = 100.0
        assert _check_select(api, torch, g, 4096)["winner"] == min(a, b)
    # every shard empty: no winner
    g, _ = _records(rng, 4, 16, [0, 0, 0, 0], False)
    dev = _check_select(api, torch, g, 16)
    assert dev["bad"] == 0 and np.all(dev["pose"] == -1)
    # a bad shard (M > 0, expert -1) is flagged, whoever wins
    g, _ = _records(rng, 3, 16, [16, 5, 9], False)
    g[1, 16 + 16] = -1.0
    assert _check_select(api, torch, g, 16)["bad"] == 1.0


def _rescale(api, torch, pairs, scores):
    ctx = api.context(0)
    M = len(scores)
    p = torch.from_numpy(np.ascontiguousarray(pairs, np.float64).reshape(-1)).cuda()
    s = torch.from_numpy(np.ascontiguousarray(scores, np.float64)).cuda() if M else None
    norm = torch.zeros(2, dtype=torch.float64, device="cuda")
    probs = torch.zeros(max(M, 1), dtype=torch.float64, device="cuda")
    contrib = torch.full((max(M, 1),), -1, dtype=torch.int32, device="cuda")
    n = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    ctx.check(ctx.lib.esacb200_test_gathered(ctx.handle, len(pairs), 0, None, None, p.data_ptr(), s.data_ptr() if M else None,
                                             M, norm.data_ptr(), probs.data_ptr(), contrib.data_ptr(), n.data_ptr()))
    k = int(n.item())
    return norm.cpu().numpy(), probs.cpu().numpy()[:M], contrib.cpu().numpy()[:k]


@pytest.mark.parametrize("world", [1, 2, 5, 64])
@pytest.mark.parametrize("M", [0, 1, 300, 1025])
def test_rescale_probs_gathered_matches_float64(api, torch, world, M):
    """The merged normalisation gmax = max_r m_r, gsum = sum_r s_r exp(m_r - gmax) in rank order, the probabilities and the
    contributing list, with neutral pairs (-1e300, 0) of empty shards among them."""
    rng = np.random.default_rng(world * 31 + M)
    scores = rng.normal(0, 3, M) + rng.uniform(-20, 20)
    pairs = np.zeros((world, 2))
    for r in range(world):
        ms = rng.normal(0, 3, int(rng.integers(1, 50))) + rng.uniform(-25, 25)
        pairs[r] = ms.max(), np.exp(ms - ms.max()).sum()
    mine = int(rng.integers(world))
    if M:
        pairs[mine] = scores.max(), np.exp(scores - scores.max()).sum()
    if world > 1:
        pairs[(mine + 1) % world] = NEUTRAL
    gmax = max(pairs[:, 0])
    gsum = 0.0
    for m, v in pairs:
        gsum += v * math.exp(m - gmax)
    p_ref = np.exp(scores - gmax) / gsum
    # keep every probability away from PROB_THRESH by more than its rounding
    near = np.abs(p_ref - O.PROB_THRESH) < 1e-9
    scores[near] += 0.01
    p_ref = np.exp(scores - gmax) / gsum
    norm, probs, contrib = _rescale(api, torch, pairs, scores)
    assert norm[0] == gmax
    assert abs(norm[1] - gsum) <= 4 * np.spacing(gsum) * world
    assert np.all(np.abs(probs - p_ref) <= 8 * np.spacing(p_ref))
    assert contrib.tolist() == np.flatnonzero(p_ref >= O.PROB_THRESH).tolist()


def test_rescale_probs_gathered_weighs_each_pair_by_its_maximum(api, torch):
    """Two ranks whose maxima differ by 3: rank 1's sum counts exp(-3) times, not once."""
    scores = np.array([0.0, -1.0, -2.0])
    pairs = np.array([[0.0, np.exp(scores).sum()], [3.0, 2.0]])
    norm, probs, _ = _rescale(api, torch, pairs, scores)
    gsum = pairs[0, 1] * np.exp(-3.0) + 2.0
    assert norm[0] == 3.0 and abs(norm[1] - gsum) < 1e-15 * gsum
    assert np.allclose(probs, np.exp(scores - 3.0) / gsum, rtol=1e-15, atol=0)


def test_hook_refuses_arguments_outside_the_kernels_contract(api, torch):
    ctx = api.context(0)
    lib = ctx.lib
    g = torch.zeros(8 + 21, dtype=torch.float64, device="cuda")
    out = torch.zeros(20, dtype=torch.float32, device="cuda")
    host = np.zeros(8 + 21)
    assert lib.esacb200_test_gathered(ctx.handle, 1, 8, None, None, None, None, 0, None, None, None, None) != 0
    assert lib.esacb200_test_gathered(ctx.handle, 0, 8, g.data_ptr(), out.data_ptr(), None, None, 0, None, None, None, None) != 0
    assert lib.esacb200_test_gathered(ctx.handle, 1, 0, g.data_ptr(), out.data_ptr(), None, None, 0, None, None, None, None) != 0
    assert lib.esacb200_test_gathered(ctx.handle, 1 << 16, 1 << 15, g.data_ptr(), out.data_ptr(), None, None, 0, None, None, None,
                                      None) != 0
    assert lib.esacb200_test_gathered(ctx.handle, 1, 8, host.ctypes.data, out.data_ptr(), None, None, 0, None, None, None,
                                      None) != 0
    assert b"host memory" in lib.esacb200_last_error(ctx.handle)
    assert lib.esacb200_test_gathered(ctx.handle, 1, 8, g.data_ptr() + 4, out.data_ptr(), None, None, 0, None, None, None,
                                      None) != 0
    pairs = torch.zeros(2, dtype=torch.float64, device="cuda")
    norm = torch.zeros(2, dtype=torch.float64, device="cuda")
    n = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.esacb200_test_gathered(ctx.handle, 1, 0, None, None, pairs.data_ptr(), None, -1, norm.data_ptr(), None, None,
                                      n.data_ptr()) != 0
    assert lib.esacb200_test_gathered(ctx.handle, 1, 0, None, None, pairs.data_ptr(), None, 4, norm.data_ptr(), None, None,
                                      n.data_ptr()) != 0
