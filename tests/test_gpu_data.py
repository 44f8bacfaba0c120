"""Device-resident image sets on the GPU (esac_b200.data): every output of a step is bitwise the reference's item path
(oracle/data_oracle.py: PIL / torchvision jitter, ToTensor, Normalize, nn.ZeroPad2d, the room offsets) for the same plan
rows, eagerly and in CUDA graphs, from both storage kinds."""
import itertools
import random
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import data
from oracle import data_oracle as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
F1_DOWN, F1_UP = float(np.nextafter(np.float32(1), np.float32(0))), float(np.nextafter(np.float32(1), np.float32(2)))
FACTORS = [0.8, 1.2, 1.0, F1_DOWN, F1_UP, 0.0, 2.5, 0.5]
PADS = [(4, -4), (-4, 4), (0, 0), (4, 4), (-4, -4), (3, -1)]


class Parts:
    """The host side of a synthetic set, what the oracle reads."""

    def __init__(self, shapes, gt_div=8, seed=0, n_attach=2):
        rng = np.random.default_rng(seed)
        self.images = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in shapes]
        N = len(shapes)
        self.poses = torch.from_numpy(rng.standard_normal((N, 4, 4)).astype(np.float32))
        self.focal = rng.uniform(400, 600, N)
        self.scenes = np.arange(N) % 3
        self.gt = []
        for H, W in shapes:
            g = torch.from_numpy(rng.standard_normal((3, H // gt_div, W // gt_div)).astype(np.float32))
            g[:, torch.from_numpy(rng.random(g.shape[1:]) < 0.3)] = 0
            self.gt.append(g)
        self.attach = {"prior": torch.from_numpy(rng.standard_normal((N, 3, 2, 3)).astype(np.float32)),
                       "gating": torch.from_numpy(rng.random((N, 5)).astype(np.float32))}
        if n_attach < 2:
            self.attach = dict(list(self.attach.items())[:n_attach])

    def set(self, storage, mean=data.ROOM_MEAN, std=data.ROOM_STD, **kw):
        return data.DeviceImageSet(self.images, self.poses, self.focal, self.scenes, gt=self.gt, attachments=self.attach,
                                   mean=mean, std=std, storage=storage, **kw)

    def expect(self, row, mean, std):
        i = int(row["image"])
        H, W = self.images[i].shape[:2]
        return {"image": O.pil_item(self.images[i], row, mean, std), "shifts": torch.tensor([row["padX"], row["padY"]], dtype=torch.int32),
                "cameras": torch.tensor([np.float32(self.focal[i]), W / 2, H / 2], dtype=torch.float32),
                "gt_poses": self.poses[i], "gt_coords": self.gt[i], "scenes": torch.tensor(self.scenes[i]),
                "indices": torch.tensor(i), **{k: v[i] for k, v in self.attach.items()}}


def _check(out, parts, rows, mean, std, what=""):
    assert int(out["status"].item()) == 0, what
    for b, row in enumerate(rows):
        want = parts.expect(row, mean, std)
        for k, v in want.items():
            got = out[k][b].cpu()
            assert got.dtype == v.dtype and torch.equal(got, v), f"{what} image {b} (row {row}): {k} differs"


def _plan(parts, ds, images, B, ops_of=None, factors_of=None):
    rows = np.zeros(len(images), api.DATA_ROW)
    for j, i in enumerate(images):
        step = j // B
        rows[j]["image"] = i
        rows[j]["padX"], rows[j]["padY"] = PADS[step % len(PADS)]
        if ops_of is not None:
            ops = ops_of(j)
            rows[j]["n_ops"] = len(ops)
            rows[j]["ops"][:len(ops)] = ops
            rows[j]["factors"][:len(ops)] = factors_of(j, len(ops))
    groups = [int(ds.group_of[images[s * B]]) for s in range(len(images) // B)]
    return data.Plan(rows, groups, B)


ORDERS = [[i for i in p if i < 3] for p in itertools.permutations(range(4))]


@pytest.mark.parametrize("storage", ["device", "pinned"])
@pytest.mark.parametrize("B", [1, 4])
def test_every_order_bitwise(storage, B):
    """The 24 ColorJitter orders with factors at and around the clip edges, pads of +-4 and 0, on 480x640, 480x642 and
    portrait images, both normalisations."""
    shapes = [(480, 640)] * 8 + [(480, 642)] * 8 + [(642, 480)] * 8
    parts = Parts(shapes, seed=B)
    for mean, std in ((data.ROOM_MEAN, data.ROOM_STD), (data.CLUSTER_MEAN, data.CLUSTER_STD)):
        ds = parts.set(storage, mean=mean, std=std)
        assert len(ds.groups) == 3
        images = list(range(24))
        plan = _plan(parts, ds, images, B, ops_of=lambda j: ORDERS[j],
                     factors_of=lambda j, n: [FACTORS[(j + 3 * k) % len(FACTORS)] for k in range(n)])
        ds.load_plan(plan)
        for s, g in enumerate(plan.groups):
            out = ds.step(g, B)
            _check(out, parts, plan.rows[s * B:(s + 1) * B], mean, std, f"{storage} B={B} step {s}")
        assert ds.state.tolist() == [24, 24]


def _snapshot(out):
    return {k: v.clone() for k, v in out.items()}


def _equal(a, b):
    return all(torch.equal(a[k], b[k]) for k in a)


def test_graph_replays_are_eager_steps_on_a_mixed_set():
    """A mixed-shape set: N replays of the per-group graphs, in plan.groups order, are bitwise N eager steps; a plan loaded
    between replays takes effect."""
    shapes = [(48, 64), (64, 48), (48, 64), (48, 66), (64, 48), (48, 66)]
    parts = Parts(shapes, seed=5)
    ds = parts.set("device")
    random.seed(2)
    torch.manual_seed(2)
    plan = ds.plan(data.ClusterDraws(len(shapes), jitter=data.cluster_jitter(True)))
    eager = []
    ds.load_plan(plan)
    for g in plan.groups:
        eager.append(_snapshot(ds.step(g)))
    for s, g in enumerate(plan.groups):
        _check(eager[s], parts, plan.rows[s:s + 1], data.ROOM_MEAN, data.ROOM_STD, f"eager step {s}")
    graphs = {}
    for g in range(len(ds.groups)):
        ds.outputs(g)
        graphs[g] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[g]):
            ds.step(g)
    ds.load_plan(plan)
    for s, g in enumerate(plan.groups):
        graphs[g].replay()
        assert _equal(_snapshot(ds.outputs(g)), eager[s]), f"replay {s}"
    # a new plan between replays
    random.seed(9)
    torch.manual_seed(9)
    plan2 = ds.plan(data.ClusterDraws(len(shapes), jitter=data.cluster_jitter(True)))
    ds.load_plan(plan2)
    for s, g in enumerate(plan2.groups[:3]):
        graphs[g].replay()
        _check(ds.outputs(g), parts, plan2.rows[s:s + 1], data.ROOM_MEAN, data.ROOM_STD, f"second plan, replay {s}")


def test_status_exhausted_and_wrong_group_leave_outputs():
    parts = Parts([(32, 40)] * 3 + [(40, 32)], seed=7)
    ds = parts.set("device")
    plan = _plan(parts, ds, [0, 1], 1)
    ds.load_plan(plan)
    ds.step(0)
    before = _snapshot(ds.step(0))
    out = ds.step(0)                       # the plan holds two rows
    assert int(out["status"].item()) == 1
    before["status"].fill_(1)
    assert _equal(_snapshot(out), before)
    assert ds.state.tolist() == [2, 2]
    ds.load_plan(_plan(parts, ds, [3], 1))   # image 3 is of group 1
    out = ds.step(0)
    assert int(out["status"].item()) == 2
    before["status"].fill_(2)
    assert _equal(_snapshot(out), before)
    assert ds.state.tolist() == [0, 1]
    out1 = ds.step(1)
    _check(out1, parts, _plan(parts, ds, [3], 1).rows, data.ROOM_MEAN, data.ROOM_STD)
    assert ds.state.tolist() == [1, 1]


def test_no_host_synchronisation():
    parts = Parts([(480, 640)] * 2, seed=1)
    ds = parts.set("device")
    ds.load_plan(_plan(parts, ds, [0, 1, 0, 1], 1))
    ds.step(0)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(int(2e9))
    ds.step(0)
    assert not stream.query(), "step waited for the device"
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ds.step(0)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))
    graph.replay()
    assert not stream.query(), "the replay waited for the device"
    torch.cuda.synchronize()
    assert int(ds.outputs(0)["status"].item()) == 0 and ds.state.tolist() == [3, 4]


def test_room_folders_with_offsets_and_empty_cells(tmp_path):
    """from_room_folders on two scenes with centres (one gray image): each step is room_dataset.py's item, offsets and
    the reset of empty ground-truth cells included, after the same draws."""
    from PIL import Image
    rng = np.random.default_rng(3)
    scenes, raw = [], []
    for s, (centre, shape) in enumerate((((1.5, -2.0, 0.25), (60, 80)), ((-3.0, 4.0, 1.0), (80, 60)))):
        d = tmp_path / f"scene{s}" / "training"
        for sub in ("rgb", "poses", "calibration", "init"):
            (d / sub).mkdir(parents=True)
        for j in range(3):
            gray = s == 1 and j == 0
            img = rng.integers(0, 256, shape if gray else shape + (3,), dtype=np.uint8)
            Image.fromarray(img).save(d / "rgb" / f"frame-{j:03d}.png")
            pose = np.eye(4)
            pose[:3, :3] = np.linalg.qr(rng.standard_normal((3, 3)))[0]
            pose[:3, 3] = rng.standard_normal(3) * 3
            np.savetxt(d / "poses" / f"frame-{j:03d}.txt", pose)
            np.savetxt(d / "calibration" / f"frame-{j:03d}.txt", [rng.uniform(500, 600)])
            g = torch.from_numpy(rng.standard_normal((3, 6, 8)).astype(np.float32) * 5)
            g[:, torch.from_numpy(rng.random((6, 8)) < 0.4)] = 0
            torch.save(g, d / "init" / f"frame-{j:03d}.dat")
            raw.append((s, d, j))
        scenes.append(f"{tmp_path / f'scene{s}'} {centre[0]} {centre[1]} {centre[2]}")
    env = tmp_path / "env_list.txt"
    env.write_text("\n".join(scenes) + "\n")
    ds = data.from_room_folders("training", imsize=48, env_list=str(env), storage="pinned")
    means = torch.tensor([[1.5, -2.0, 0.25], [-3.0, 4.0, 1.0]])
    random.seed(4)
    torch.manual_seed(4)
    plan = ds.plan(data.RoomDraws(ds.scene_counts))
    ds.load_plan(plan)
    for step, g in enumerate(plan.groups[:12]):
        out = ds.step(g)
        row = plan.rows[step]
        s, d, j = raw[int(row["image"])]
        name = f"frame-{j:03d}"
        a = np.asarray(Image.open(d / "rgb" / f"{name}.png"))
        if a.ndim == 2:
            a = np.stack([a] * 3, -1)
        scale = 48 / min(a.shape[:2])
        from torchvision import transforms
        resized = np.asarray(transforms.Resize(48)(transforms.ToPILImage()(a)))
        pose, coords = O.room_offset(torch.from_numpy(np.loadtxt(d / "poses" / f"{name}.txt")).float(),
                                     torch.load(d / "init" / f"{name}.dat"), means[s], s, 2)
        f = float(np.loadtxt(d / "calibration" / f"{name}.txt")) * scale
        H, W = resized.shape[:2]
        assert int(out["status"].item()) == 0
        assert torch.equal(out["image"][0].cpu(), O.pil_item(resized, row, data.ROOM_MEAN, data.ROOM_STD)), step
        assert torch.equal(out["gt_poses"][0].cpu(), pose), step
        assert torch.equal(out["gt_coords"][0].cpu(), coords), step
        assert torch.equal(out["cameras"][0].cpu(), torch.tensor([np.float32(f), W / 2, H / 2])), step
        assert int(out["scenes"][0]) == s and int(out["indices"][0]) == int(row["image"])
        assert bool((coords.abs().sum(0) == 0).any())


def test_example_runs_with_check():
    r = subprocess.run([sys.executable, str(ROOT / "examples" / "init_expert_step_device_data_synthetic.py"),
                        "--iterations", "6", "--check"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "check ok" in r.stdout
