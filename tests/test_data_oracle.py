"""The host side of esac_b200.data, without a GPU: the numpy restatement the kernels state equals PIL / torchvision's item
path, and the planner's rows are the reference loop's draws."""
import itertools
import random

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision.transforms import functional as F

import esac_b200.api as api
from esac_b200 import data
from oracle import data_oracle as O


def _row(ops, factors, padX=0, padY=0, image=0):
    r = np.zeros((), api.DATA_ROW)
    r["image"], r["padX"], r["padY"], r["n_ops"] = image, padX, padY, len(ops)
    r["ops"][:len(ops)] = ops
    r["factors"][:len(ops)] = factors
    return r


@pytest.mark.parametrize("fn_idx", list(itertools.permutations(range(4))), ids=lambda p: "".join(map(str, p)))
def test_restatement_is_pil_for_every_order(fn_idx):
    """ColorJitter's 24 orders (hue, index 3, off as in the reference's jitter) with factors from its uniform_ draws."""
    rng = np.random.default_rng(sum(v * 4 ** i for i, v in enumerate(fn_idx)))
    torch.manual_seed(len(fn_idx) * 7 + fn_idx[0])
    for trial in range(6):
        image = rng.integers(0, 256, (23, 31, 3), dtype=np.uint8)
        factors = {0: float(torch.empty(1).uniform_(0.8, 1.2)), 1: float(torch.empty(1).uniform_(0.8, 1.2)),
                   2: [0.0, float(torch.empty(1).uniform_(0, 1)), float(torch.empty(1).uniform_(0.8, 1.2))][trial % 3]}
        ops = [i for i in fn_idx if i < 3]
        row = _row(ops, [factors[o] for o in ops], padX=trial - 3, padY=2 - trial)
        for mean, std in ((data.ROOM_MEAN, data.ROOM_STD), (data.CLUSTER_MEAN, data.CLUSTER_STD)):
            want = O.pil_item(image, row, mean, std).numpy()
            np.testing.assert_array_equal(O.restate_item(image, row, mean, std), want)


def _nextafter(x, d):
    return float(np.nextafter(np.float32(x), np.float32(d)))


@pytest.mark.parametrize("f", [0.0, 1.0, 0.8, 1.2, _nextafter(1, 0), _nextafter(1, 2), 0.5, 1.5, -0.25])
def test_blend_over_all_byte_pairs(f):
    a, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    want = np.asarray(Image.blend(Image.fromarray(a), Image.fromarray(b), f))
    np.testing.assert_array_equal(O.blend(a, b, f), want)


@pytest.mark.parametrize("mean, std", [(data.ROOM_MEAN, data.ROOM_STD), (data.CLUSTER_MEAN, data.CLUSTER_STD)])
def test_normalisation_over_all_values(mean, std):
    u = np.repeat(np.arange(256, dtype=np.uint8)[:, None, None], 3, -1)   # [256,1,3]
    want = F.normalize(F.to_tensor(Image.fromarray(u)), [mean] * 3, [std] * 3).numpy()
    np.testing.assert_array_equal(O.normalize(u, mean, std), want)


def test_luma_and_contrast_grey_are_pil():
    rng = np.random.default_rng(5)
    for shape in ((17, 29, 3), (480, 640, 3)):
        image = rng.integers(0, 256, shape, dtype=np.uint8)
        np.testing.assert_array_equal(O.luma(image), np.asarray(Image.fromarray(image).convert("L")))
        for f in (0.8, 1.2, 0.0):
            np.testing.assert_array_equal(O.jitter(image, [(O.CONTRAST, f)]),
                                          np.asarray(F.adjust_contrast(Image.fromarray(image), f)))


def _seeded(seed):
    random.seed(seed)
    torch.manual_seed(seed)


def _check_rows(plan, drawn, jitter=None):
    assert len(plan.rows) >= len(drawn)
    for step, (row, (image, padX, padY, params)) in enumerate(zip(plan.rows, drawn)):
        assert (int(row["image"]), int(row["padX"]), int(row["padY"])) == (image, padX, padY), step
        if params is None:
            assert row["n_ops"] == 0
            continue
        fn_idx, b, c, s, _ = params
        factor = {0: b, 1: c, 2: s}
        ops = [int(i) for i in fn_idx if int(i) < 3 and factor[int(i)] is not None]
        assert list(row["ops"][:row["n_ops"]]) == ops, step
        assert list(row["factors"][:row["n_ops"]]) == [np.float32(factor[o]) for o in ops], step


@pytest.mark.parametrize("scene", [-1, 1])
def test_planner_draws_the_room_loop(scene):
    counts = [5, 7, 3]
    _seeded(11)
    drawn = O.reference_loop("room", 40, counts=counts, scene=scene)
    _seeded(11)
    group_of = np.zeros(sum(counts), np.int32)
    plan = data.make_plan(data.RoomDraws(counts, scene=scene), group_of)
    assert plan.groups == [0] * len(plan.rows) and len(plan.rows) == (1000 if scene < 0 else counts[scene])
    _check_rows(plan, drawn)


def test_planner_draws_the_room_test_order():
    counts = [4, 2]
    drawn = O.reference_loop("room", 6, counts=counts, training=False, shuffle=False, shift=False)
    plan = data.make_plan(data.RoomDraws(counts, training=False), np.zeros(6, np.int32), shuffle=False, shift=False)
    assert [int(r["image"]) for r in plan.rows] == list(range(6))
    _check_rows(plan, drawn)


@pytest.mark.parametrize("cluster", [True, False])
def test_planner_draws_the_cluster_loop(cluster):
    n = 9
    probs = torch.softmax(torch.arange(n, dtype=torch.float32) * 0.3, 0) if cluster else None
    jitter = data.cluster_jitter(True)
    _seeded(3)
    drawn = O.reference_loop("cluster", n, n=n, probs=probs, jitter=jitter)
    _seeded(3)
    plan = data.make_plan(data.ClusterDraws(n, probs=probs, jitter=jitter), np.zeros(n, np.int32))
    _check_rows(plan, drawn, jitter)
    assert {int(r["n_ops"]) for r in plan.rows} == {3}


def test_planner_draws_the_cluster_test_order():
    n = 5
    jitter = data.cluster_jitter(False)
    _seeded(4)
    drawn = O.reference_loop("cluster", n, n=n, jitter=jitter, shuffle=False, shift=False)
    _seeded(4)
    plan = data.make_plan(data.ClusterDraws(n, jitter=jitter), np.zeros(n, np.int32), shuffle=False, shift=False)
    assert [int(r["image"]) for r in plan.rows] == list(range(n))
    assert all(int(r["n_ops"]) == 1 and r["ops"][0] == api.DATA_SATURATION and r["factors"][0] == 0 for r in plan.rows)
    _check_rows(plan, drawn, jitter)


def test_planner_batches_share_a_shift_and_a_group():
    _seeded(8)
    plan = data.make_plan(data.ClusterDraws(8), np.array([0, 0, 1, 1, 0, 0, 1, 1], np.int32), batch=2, shuffle=False)
    assert plan.groups == [0, 1, 0, 1] and plan.batch == 2
    assert all(plan.rows["padX"][0::2] == plan.rows["padX"][1::2])
    with pytest.raises(ValueError, match="mixes shape groups"):
        data.make_plan(data.ClusterDraws(4), np.array([0, 1, 0, 1], np.int32), batch=2, shuffle=False)

