"""BASELINE.json's full size (480x640, subSampling 1, 256 hypotheses x 7 experts): size-independent properties and
spot checks against the C oracle restatement (fast enough for a handful of hypotheses at this size)."""
import numpy as np
import pytest

from esac_b200.synth import make_scene, pose_error
from oracle.build import c_score

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    import esac_b200.api as api
    api.context().set_option("fixed_seed", 1)
    return api


@pytest.fixture(scope="module")
def scene():
    return make_scene(E=7, H=480, W=640, M=256, sub=1, seed=0, per_expert=True, active_only=False)


def test_known_answer_at_full_resolution(api):
    sc = make_scene(E=2, H=480, W=640, M=64, sub=1, seed=5, outlier_frac=0.3, noise=0.0)
    out = np.zeros((4, 4), np.float32)
    api.set_seed(1)
    e = api.forward(sc.coords, sc.assign, out, *sc.params)
    rot, trans = pose_error(out, sc.gt_pose)
    assert e == sc.gt_expert and rot < 2e-3 and trans < 2e-4  # float32 coordinates limit the recovery


def test_scores_spot_check_against_c_oracle(api, scene):
    sc = scene
    api.set_seed(11)
    out = np.zeros((4, 4), np.float32)
    api.forward(sc.coords, sc.assign, out, *sc.params)
    hy = api.last_hypotheses()
    idx = np.array([0, 100, 300, 511, 700, 1000, 1500, 1791])
    ref, _ = c_score(sc.coords, sc.assign[idx], hy["poses"][idx], *sc.params)
    assert np.abs(ref - hy["scores"][idx]).max() < 1e-4


def test_scores_are_permutation_invariant_and_deterministic(api, scene):
    sc = scene
    rng = np.random.default_rng(0)
    M = len(sc.assign)
    poses = np.zeros((M, 6))
    poses[:, :3] = rng.normal(0, 0.3, (M, 3))
    poses[:, 3:] = rng.normal(0, 2.0, (M, 3))
    s0 = api.score_poses(sc.coords, sc.assign, poses, *sc.params)
    s1 = api.score_poses(sc.coords, sc.assign, poses, *sc.params)
    assert np.array_equal(s0, s1)  # bit-reproducible (fixed-order reductions)
    perm = rng.permutation(M)
    s2 = api.score_poses(sc.coords, sc.assign[perm], poses[perm], *sc.params)
    assert np.abs(s2 - s0[perm]).max() < 1e-9  # chunking changes, per-hypothesis arithmetic does not


def test_score_scales_linearly_with_alpha(api, scene):
    sc = scene
    rng = np.random.default_rng(1)
    M = 64
    poses = np.zeros((M, 6))
    poses[:, :3] = rng.normal(0, 0.2, (M, 3))
    poses[:, 3:] = rng.normal(0, 1.0, (M, 3)) + [0, 0, 2]
    a = list(sc.params)
    s1 = api.score_poses(sc.coords, sc.assign[:M], poses, *a)
    a[6] = 200.0  # inlierAlpha
    s2 = api.score_poses(sc.coords, sc.assign[:M], poses, *a)
    assert np.abs(s2 - 2 * s1).max() < 1e-5
    assert s1.min() >= 0 and s1.max() <= 100.0


def test_forward_is_reproducible_and_winner_is_local_argmax(api, scene):
    sc = scene
    outs = []
    for _ in range(2):
        api.set_seed(21)
        out = np.zeros((4, 4), np.float32)
        e = api.forward(sc.coords, sc.assign, out, *sc.params)
        outs.append((e, out.copy(), api.last_hypotheses()["scores"], api.last_stats()["winner"]))
    assert outs[0][0] == outs[1][0] and np.array_equal(outs[0][1], outs[1][1]) and np.array_equal(outs[0][2], outs[1][2])
    assert outs[0][3] == int(np.argmax(outs[0][2]))
    assert outs[0][0] == sc.gt_expert
    rot, trans = pose_error(outs[0][1], sc.gt_pose)
    assert rot < 0.1 and trans < 0.01


@pytest.mark.parametrize("kw", [dict(E=7, M=256, per_expert=True), dict(E=3, M=200), dict(E=2, M=64, gt_mass=1.0)])
def test_split_upload_of_host_maps_changes_nothing(api, kw):
    """Host maps >= 4 MB are uploaded in two halves with the first half's experts sampled under the second copy
    (lanes dealt by expert).  Scores, sampled sets, winner and pose must equal the plain path, CPU tensors and CUDA tensors
    alike; an expert half without any hypothesis (gt_mass = 1) is an empty lane."""
    import torch
    sc = make_scene(H=480, W=640, sub=1, seed=31, active_only=False, **kw)
    ctx = api.context()
    res = {}
    for mode in ("split", "plain", "cuda"):
        ctx.set_option("upload_split", 1 if mode == "split" else 0)
        api.set_seed(77)
        if mode == "cuda":
            out = torch.zeros(4, 4, device="cuda")
            e = api.forward(torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda(), out, *sc.params)
            out = out.cpu().numpy()
        else:
            out = np.zeros((4, 4), np.float32)
            e = api.forward(torch.from_numpy(sc.coords).pin_memory(), torch.from_numpy(sc.assign), torch.from_numpy(out), *sc.params)
        hy = api.last_hypotheses()
        res[mode] = (e, out.copy(), hy["scores"].copy(), hy["cells"].copy(), hy["tries"].copy())
    ctx.set_option("upload_split", 1)
    for mode in ("plain", "cuda"):
        assert res["split"][0] == res[mode][0]
        assert np.array_equal(res["split"][1], res[mode][1])
        assert np.array_equal(res["split"][3], res[mode][3]) and np.array_equal(res["split"][4], res[mode][4])
        assert np.array_equal(res["split"][2], res[mode][2])


def test_refinement_code_paths_agree_at_full_resolution(api):
    """The refinement kernel has three ways to walk a CTA's share of the map's 32-cell mask words: cells + inlier list in
    shared memory (share <= 96 words), inlier list in global scratch (<= 2048 words), and predicated passes over all cells
    (larger shares, or refine_compact = 0).  Forcing the group size selects each of them at 480x640 (9600 words); the largest
    group is every co-resident CTA, as last_stats() reports it.  Rounds and inlier counts must be identical and the poses equal
    up to the summation order (1e-9)."""
    sc = make_scene(E=1, H=480, W=640, M=6, sub=1, seed=21, outlier_frac=0.4)
    import cv2
    rng = np.random.default_rng(21)
    T = np.linalg.inv(sc.gt_pose.astype(np.float64))
    poses6 = np.zeros((len(sc.assign), 6))
    for h in range(len(sc.assign)):
        dR, _ = cv2.Rodrigues(rng.normal(0, 0.003, 3))
        poses6[h, :3] = cv2.Rodrigues(dR @ T[:3, :3])[0].ravel()
        poses6[h, 3:] = dR @ T[:3, 3] + rng.normal(0, 0.01, 3)
    words = (480 * 640 + 31) // 32
    share = lambda g: -(-words // g)                                 # noqa: E731
    ctx = api.context()
    outs = {}

    def run(grp, compact):
        ctx.set_option("refine_group", grp)
        ctx.set_option("refine_compact", compact)
        res = api.refine_poses(sc.coords, sc.assign, poses6, sc.shiftX, sc.shiftY, sc.f, sc.ppx, sc.ppy, sc.tau, sc.max_reproj, sc.sub)
        return res, api.last_stats()["refine_group"]

    try:
        res, g_max = run(1 << 20, 1)
        assert share(g_max) <= 96, (g_max, share(g_max))            # shared-memory lists need every co-resident CTA
        outs["shared-list"] = res
        g_list = -(-words // 1024)                                      # ~1024 words per CTA: global lists
        g_all = 2                                                       # 4800 words per CTA: no lists
        assert 96 < share(g_list) <= 2048 and share(g_all) > 2048
        for walk, grp, compact in (("global-list", g_list, 1), ("all-cells", g_all, 1), ("cached-all-cells", g_max, 0),
                                   ("all-cells-uncompacted", g_list, 0)):
            outs[walk], g = run(grp, compact)
            assert g == grp, (walk, g, grp)
    finally:
        ctx.set_option("refine_group", 0)
        ctx.set_option("refine_compact", 1)
    base = outs["shared-list"]
    assert base[1].max() >= 1 and base[2].min() > 1000
    for walk, o in outs.items():
        assert o[1].tolist() == base[1].tolist(), walk
        assert o[2].tolist() == base[2].tolist(), walk
        assert np.abs(o[0] - base[0]).max() < 1e-9, walk
