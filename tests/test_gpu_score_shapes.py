"""Every scoring launch shape against the float64 reference (oracle/score_fp64.py), not only the ones the heuristics pick.

plan_and_prep (capi_pipeline.cu) picks ppt (cells per thread, tile = 256 * ppt cells), hc (hypotheses per chunk) and one of three
load paths from `vec_ok = N % a == 0 and base % (4 a) == 0`, a = 4 if ppt >= 4 else 2:
  TMA bulk copies when vec_ok and ppt >= 4; vector __ldg when vec_ok and ppt == 2; scalar loads otherwise,
each with a ragged-tail form when N % tile != 0.  The options score_ppt / score_hc force the shape; the test ids name the
load path that this rule derives, and every test asserts the ppt that ran.

Single-cell probes: the maps are built so that at known poses every cell has a prescribed reprojection error, all of them
beyond maxReproj except one probe cell per expert plane, whose error sits within a few pixels of tau where the soft-inlier
weight is steepest.  With alpha = N a hypothesis' score is its probe's weight (the other cells add N e^-45), so one cell
read wrongly or a pixel centre off by one pixel moves a score by >= 1e-2, against a tolerance of 1e-5."""
import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error, rodrigues
from oracle import score_fp64

pytestmark = pytest.mark.gpu

TPS = (512, 1024, 2048)
PPTS = (2, 4, 8)
HCS = (1, 3, 5, 33, 64)
PROBE_TOL = 1e-5
SCORE_TOL = 1e-4           # BASELINE.json's score tolerance (alpha = 100)
ORDER_TOL = 1e-5           # two launch shapes of one scene differ only in the summation order


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


def load_path(N: int, ptr: int, ppt: int) -> str:
    """The load path plan_and_prep / launch_score pick (capi_pipeline.cu, score.cu), plus '-tail' for a ragged last tile."""
    a = 4 if ppt >= 4 else 2
    vec_ok = N % a == 0 and ptr % (4 * a) == 0
    path = "tma" if vec_ok and ppt >= 4 else ("vec" if vec_ok else "scalar")
    return path + ("-tail" if N % (256 * ppt) else "")


def score_forced(api, coords, assign, poses, params, ppt, hc):
    ctx = api.context()
    ctx.set_option("score_ppt", ppt)
    ctx.set_option("score_hc", hc)
    try:
        got = api.score_poses(coords, assign, poses, *params)
        assert api.last_stats()["score_ppt"] == ppt
    finally:
        ctx.set_option("score_ppt", 0)
        ctx.set_option("score_hc", 0)
    return got


def misaligned(t):
    """A contiguous CUDA copy of `t` whose base is 4 bytes past a 16-byte boundary (N % 4 may still be 0)."""
    import torch
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device="cuda")
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


# ---- probe maps --------------------------------------------------------------------------------------------------------
def probe_cells(H, W):
    """First and last cell, last cell of a row, both sides of every tile boundary k*TP (first and last boundary), the last
    cell of the last whole tile, and four consecutive cells = 0, 1, 2, 3 (mod 4) in the middle of the map."""
    N = H * W
    cells = {0, N - 1, W - 1, (H // 2) * W + W - 1}
    for tp in TPS:
        for k in (1, N // tp):
            if 0 < k * tp < N:
                cells |= {k * tp - 1, k * tp}
    m = (N // 2) & ~3
    cells |= {m, m + 1, m + 2, m + 3}
    return sorted(c for c in cells if 0 <= c < N)


KINDS = ("near", "mirrored", "world", "millimetres")


def probe_scene(H, W, sub, shiftX, shiftY, seed):
    """Probe maps at H x W: one plane per probe cell plus an expert without hypotheses, 1..7 perturbed poses per plane in a
    shuffled assignment, depth kinds cycling through positive, negative (every cell mirrored through the principal point:
    same projection), world-scale (700 m from the origin) and millimetre units."""
    rng = np.random.default_rng(seed)
    f, tau, beta, max_reproj = 525.0, 10.0, 0.5, 100.0
    ppx, ppy = W * sub / 2.0, H * sub / 2.0
    N = H * W
    probes = probe_cells(H, W)
    E = len(probes) + 1
    empty = 2                                                    # a gap in the chunk table
    px, py = score_fp64.pixel_centres(H, W, sub, shiftX, shiftY)
    px, py = px.reshape(-1), py.reshape(-1)
    coords = np.zeros((E, 3, N), np.float32)
    assign, poses = [], []
    counts = (2, 3, 5, 1, 7, 4, 6)
    for i, cell in enumerate(probes):
        e = i if i < empty else i + 1
        kind = KINDS[i % len(KINDS)]
        scale = 1000.0 if kind == "millimetres" else 1.0
        R = rodrigues(rng.normal(0, 0.3, 3))
        C = (700.0 if kind == "world" else 0.0) + rng.uniform(-1, 1, 3) * scale
        t = -R @ C
        # every cell 130..400 px off its pixel centre, the probe tau + (-3..3) px off, in varying directions
        ang = rng.uniform(0, 2 * np.pi, N)
        mag = rng.uniform(130.0, 400.0, N)
        ang[cell] = np.pi / 4 + (i % 4) * np.pi / 2 + rng.uniform(-0.3, 0.3)
        mag[cell] = tau + rng.uniform(-3.0, 3.0)
        u, v = px + mag * np.cos(ang), py + mag * np.sin(ang)
        depth = rng.uniform(1.0, 5.0, N) * scale * (2.0 if kind == "world" else 1.0)
        if kind == "mirrored":
            depth = -depth
        cam = np.stack([(u - ppx) / f * depth, (v - ppy) / f * depth, depth])
        coords[e] = (R.T @ (cam - t[:, None])).astype(np.float32)
        for _ in range(counts[i % len(counts)]):
            dR = rodrigues(rng.normal(0, 0.001, 3))             # a rotation about the camera centre: ~0.5 px
            poses.append(np.concatenate([_rvec(dR @ R), dR @ t]))
            assign.append(e)
    order = rng.permutation(len(assign))
    assign = np.array(assign, np.int64)[order]
    poses = np.array(poses)[order]
    coords = coords.reshape(E, 3, H, W)
    params = (shiftX, shiftY, f, ppx, ppy, tau, float(N), beta, max_reproj, sub)   # alpha = N
    return coords, assign, poses, params


def _rvec(R):
    th = np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return w * (th / (2 * np.sin(th))) if th > 1e-12 else 0.5 * w


PROBE_SHAPES = {                          # name: (H, W, sub, shiftX, shiftY, misaligned view)
    "480x640": (480, 640, 1, 0, 0, False),           # whole tiles for every ppt
    "480x640-offset": (480, 640, 1, 3, -5, True),    # N % 4 == 0 but a misaligned base: scalar loads, whole tiles
    "120x160": (120, 160, 3, 3, -5, False),          # ragged tiles for every ppt
    "60x80": (60, 80, 8, 3, -5, False),
    "61x81": (61, 81, 3, 0, 0, False),               # odd N: scalar loads, ragged
    "60x80-offset": (60, 80, 8, 0, 0, True),         # misaligned: scalar loads with ppt >= 4, ragged
}
_probe_cache = {}


def _probe(name):
    if name not in _probe_cache:
        H, W, sub, sx, sy, off = PROBE_SHAPES[name]
        coords, assign, poses, params = probe_scene(H, W, sub, sx, sy, seed=H + W + sub)
        ref, _ = score_fp64.score(coords, assign, poses, *params)
        _probe_cache[name] = (coords, assign, poses, params, ref, off)
    return _probe_cache[name]


def _probe_ids():
    out = []
    for name, (H, W, sub, sx, sy, off) in PROBE_SHAPES.items():
        ptr = 4 if off else 0
        for ppt in PPTS:
            path = load_path(H * W, ptr, ppt)
            out.append(pytest.param(name, ppt, path, id=f"{name}-sub{sub}-ppt{ppt}-{path}"))
    return out


def test_probe_maps_put_every_probe_on_the_steep_part_of_the_weight():
    """The probe construction itself (CPU): each hypothesis' score is one probe weight well inside (0, 1), and moving every
    pixel centre by one pixel moves the scores by >= 1e-2 -- the size of mistake the probes exist to catch."""
    coords, assign, poses, params, ref, _ = _probe("61x81")
    assert 0.01 < ref.min() and ref.max() < 0.99
    shifted = list(params)
    shifted[0] -= 1
    shifted[1] -= 1
    ref1, _ = score_fp64.score(coords, assign, poses, *shifted)
    assert np.abs(ref1 - ref).max() > 1e-2


@pytest.mark.parametrize("name,ppt,path", _probe_ids())
def test_single_cell_probes_every_launch_shape(api, name, ppt, path):
    import torch
    coords, assign, poses, params, ref, off = _probe(name)
    assert 0.01 < ref.min() and ref.max() < 0.99
    t = torch.from_numpy(coords).cuda()
    if off:
        t = misaligned(t)
    a = torch.from_numpy(assign).cuda()
    N = coords.shape[2] * coords.shape[3]
    assert load_path(N, t.data_ptr(), ppt) == path
    for hc in HCS:
        got = score_forced(api, t, a, poses, params, ppt, hc)
        bad = np.abs(got - ref)
        assert bad.max() < PROBE_TOL, (hc, int(bad.argmax()), got[bad.argmax()], ref[bad.argmax()])


# ---- dense scenes --------------------------------------------------------------------------------------------------------
def _dense_poses(sc, rng, M):
    """Half near the ground truth (many cells close to tau), half arbitrary (cells behind the camera, far off)."""
    T = np.linalg.inv(sc.gt_pose.astype(np.float64))
    poses = np.zeros((M, 6))
    for h in range(M):
        if h % 2 == 0:
            dR = rodrigues(rng.normal(0, 0.01, 3))
            poses[h, :3] = _rvec(dR @ T[:3, :3])
            poses[h, 3:] = dR @ T[:3, 3] + rng.normal(0, 0.03, 3)
        else:
            poses[h, :3] = rng.normal(0, 0.5, 3)
            poses[h, 3:] = T[:3, 3] + rng.normal(0, 2.0, 3)
    return poses


@pytest.mark.parametrize("H,W,sub", [(480, 640, 1), (120, 160, 4)])
def test_load_paths_are_bitwise_identical(api, H, W, sub):
    """TMA, vector and scalar loads bring the same values into the same registers, and the per-cell arithmetic and the
    summation order do not depend on the path: with ppt and hc fixed, an aligned map and the same map as a misaligned view
    score bit for bit alike."""
    import torch
    sc = make_scene(E=3, H=H, W=W, M=40, sub=sub, seed=H + 1, shiftX=2, shiftY=-1)
    poses = _dense_poses(sc, np.random.default_rng(H), len(sc.assign))
    a = torch.from_numpy(sc.assign).cuda()
    t = torch.from_numpy(sc.coords).cuda()
    tm = misaligned(t)
    N = H * W
    for ppt in PPTS:
        p_al, p_mis = load_path(N, t.data_ptr(), ppt), load_path(N, tm.data_ptr(), ppt)
        assert p_al.split("-")[0] in ("tma", "vec") and p_mis.split("-")[0] == "scalar"
        s_al = score_forced(api, t, a, poses, sc.params, ppt, 16)
        s_mis = score_forced(api, tm, a, poses, sc.params, ppt, 16)
        assert np.array_equal(s_al, s_mis), (ppt, p_al, p_mis, np.abs(s_al - s_mis).max())
        assert s_al.max() > 1.0                                   # some poses do have inliers


DENSE = {
    "120x160-sub4": dict(E=3, H=120, W=160, M=36, sub=4, seed=31, shiftX=3, shiftY=-5),
    "61x81-sub3-world": dict(E=2, H=61, W=81, M=30, sub=3, seed=32, world_offset=700.0),
    "60x80-sub8-noisy": dict(E=4, H=60, W=80, M=45, sub=8, seed=33, noise=0.05, outlier_frac=0.3),
}


@pytest.mark.parametrize("name", list(DENSE))
def test_dense_scores_every_launch_shape(api, name):
    """Random scenes and poses under every forced (ppt, hc): within BASELINE's 1e-4 of the fp64 reference, and within 1e-5
    of each other (only the order of the partial sums differs between shapes)."""
    import torch
    sc = make_scene(**DENSE[name])
    poses = _dense_poses(sc, np.random.default_rng(DENSE[name]["seed"]), len(sc.assign))
    ref, _ = score_fp64.score(sc.coords, sc.assign, poses, *sc.params)
    assert ref.max() > 5.0
    t = torch.from_numpy(sc.coords).cuda()
    a = torch.from_numpy(sc.assign).cuda()
    first = None
    for ppt in PPTS:
        for hc in HCS:
            got = score_forced(api, t, a, poses, sc.params, ppt, hc)
            assert np.abs(got - ref).max() < SCORE_TOL, (ppt, hc, np.abs(got - ref).max())
            if first is None:
                first = got
            assert np.abs(got - first).max() < ORDER_TOL, (ppt, hc, np.abs(got - first).max())


# ---- the camera-centre case ---------------------------------------------------------------------------------------------
def test_hypotheses_on_an_all_zero_plane_never_outrank_real_ones(api):
    """An expert whose plane is all zeros (train_esac.py leaves inactive experts at zero) gives up sampling with the zero
    pose, so every cell of its plane sits at the camera centre.  Such a cell scores as maxReproj (DESIGN.md §2), so these
    hypotheses score ~0: they must neither win the forward nor outrank any real hypothesis."""
    sc = make_scene(E=2, H=30, W=40, M=16, sub=8, seed=15, outlier_frac=0.3)
    zero_e = 1 - sc.gt_expert
    sc.coords[zero_e] = 0.0
    assign = np.array([sc.gt_expert, zero_e] * 8, np.int64)
    api.set_option("max_tries", 3000)
    try:
        api.set_seed(1)
        out = np.zeros((4, 4), np.float32)
        e = api.forward(sc.coords, assign, out, *sc.params)
        hy = api.last_hypotheses()
        st = api.last_stats()
    finally:
        api.set_option("max_tries", 1000000)
    on_zero = assign == zero_e
    assert hy["tries"][on_zero].tolist() == [3000] * 8 and np.all(hy["poses"][on_zero] == 0)
    assert hy["scores"][on_zero].max() < hy["scores"][~on_zero].min(), (hy["scores"][on_zero], hy["scores"][~on_zero])
    assert e == sc.gt_expert and assign[st["winner"]] == sc.gt_expert
    rot, trans = pose_error(out, sc.gt_pose)
    assert rot < 1.0 and trans < 0.05
    # the rule itself: the zero pose on the zero plane = every cell at err = maxReproj
    got = api.score_poses(sc.coords, np.array([zero_e], np.int64), np.zeros((1, 6)), *sc.params)
    want = sc.alpha * score_fp64.soft_inlier_weights(np.array([sc.max_reproj]), sc.tau, sc.beta)[0]
    assert abs(got[0] - want) < 1e-4 * want, (got[0], want)     # fp32 exp2 of an exponent ~65
