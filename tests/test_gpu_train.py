"""train_esac.py on the device in one command (python -m esac_b200.train): on synthetic training environments written
under tmp_path -- a room environment of three scenes with images of two shapes, and a clustered environment of portrait
and landscape images -- the model file and every log line equal those of an eager twin of the reference's loop, written
here: the same plans and seeds, networks.Expert / networks.Gating, api.assign_hypotheses, eager esac_loss, the same Adam
settings, and a forward, backward and step of only the experts with hypotheses."""
import os
import random
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api
from esac_b200 import train
from esac_b200.autograd import esac_loss
from esac_b200.compat import OUTPUT_SUBSAMPLE
from esac_b200.data import from_cluster_folder, from_room_folders
from esac_b200.experts import ExpertStack, prediction_size
from esac_b200.gating_net import GatingNet
from esac_b200.networks import Expert, Gating
from oracle import expert_oracle as XO
from oracle import gating_oracle as GO

ROOT = Path(__file__).resolve().parents[1]
pytestmark = pytest.mark.gpu


def write_environment(root: Path, scenes: int, shapes, seed: int):
    """Scene folders with training/{rgb,poses,calibration,init} and test/{rgb,poses,calibration} files, and env_list.txt."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    names = []
    for s in range(scenes):
        for part in ("training", "test"):
            base = root / f"scene{s}" / part
            subs = ("rgb", "poses", "calibration") + (("init",) if part == "training" else ())
            for sub in subs:
                (base / sub).mkdir(parents=True)
            for j, (h, w) in enumerate(shapes):
                low = rng.random((h // 8, w // 8, 3))
                img = np.kron(low, np.ones((8, 8, 1))) * 200 + rng.random((h, w, 3)) * 40
                Image.fromarray(img.clip(0, 255).astype(np.uint8)).save(base / "rgb" / f"frame-{j:06d}.color.png")
                pose = np.eye(4)
                pose[:3, 3] = rng.normal(size=3)
                np.savetxt(base / "poses" / f"frame-{j:06d}.pose.txt", pose)
                np.savetxt(base / "calibration" / f"frame-{j:06d}.calibration.txt", [525.0 + 10 * j])
                if part == "training":   # the maps of the images as the data set resizes them (shorter side 480)
                    H, W = (480, 480 * w // h) if h <= w else (480 * h // w, 480)
                    coords = torch.from_numpy(rng.normal(size=(3,) + prediction_size(H, W)).astype(np.float32))
                    torch.save(coords, base / "init" / f"frame-{j:06d}.dat")
        names.append(str(root / f"scene{s}"))
    (root / "env_list.txt").write_text("".join(n + "\n" for n in names))


def write_networks(root: Path, E: int, capacity: int, session: str, seed: int):
    """gating_<session>.net, expert_e<i>_<session>.net and expert_e<i>_<session>_refined.net (other weights)."""
    torch.save(GO.kaiming_state_dict(seed, E, capacity), root / f"gating_{session}.net")
    for e in range(E):
        mean = (0.3 * e, -0.5, 2.0 + 0.2 * e)
        torch.save(XO.kaiming_state_dict(seed + 1 + e, mean=mean), root / f"expert_e{e}_{session}.net")
        torch.save(XO.kaiming_state_dict(seed + 50 + e, mean=mean), root / f"expert_e{e}_{session}_refined.net")


def run(cwd: Path, module: str, *args):
    env = dict(os.environ, PYTHONPATH=str(ROOT) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", module, *args], cwd=cwd, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


class Chdir:
    def __init__(self, path):
        self.path, self.prev = path, None

    def __enter__(self):
        self.prev = os.getcwd()
        os.chdir(self.path)

    def __exit__(self, *exc):
        os.chdir(self.prev)


def environment(cwd: Path, opt):
    """The command's training set, draws, networks and optimisers for `opt`."""
    clustered = opt.clusters >= 0
    with Chdir(cwd):
        ds = from_cluster_folder("training", training=True) if clustered else from_room_folders("training", training=True)
        E, capacity = (opt.clusters, 2) if clustered else (len(ds.scene_counts), 1)
        gating, experts = train.load_networks(opt, E, capacity, "cuda")
    draws = train.training_draws(ds, clustered)
    gating_opt, expert_opts = train.optimizers(opt, gating, experts)
    return ds, draws, gating, experts, gating_opt, expert_opts


def deterministic():
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False


def twin(cwd: Path, argv):
    """The reference's loop (train_esac.py:95-188) on the library's pieces, eagerly: returns the saved state dicts and the
    log lines."""
    opt = train.options(argv)
    ds, draws, gating, experts, gating_opt, expert_opts = environment(cwd, opt)
    E, M = len(experts), opt.hypotheses
    deterministic()
    random.seed(opt.seed)
    torch.manual_seed(opt.seed)
    api.context().set_option("fixed_seed", 0)
    api.set_seed(opt.seed)
    lines, it = [], 0
    for _ in range(train.epochs(opt.iterations, len(draws))):
        plan = train.epoch_plan(ds, draws)
        ds.load_plan(plan)
        for g in plan.groups:
            out = ds.step(g)
            image = out["image"]
            log_p = gating(image)
            probs = torch.exp(log_p).detach()
            e_hyps, hist = api.assign_hypotheses(probs, M, opt.seed + it, maxExperts=opt.maxexperts,
                                                 expertSelection=opt.expertselection)
            counts = hist[0].tolist()
            active = [e for e in range(E) if counts[e] > 0]
            prediction = torch.zeros((E, 3) + prediction_size(*image.shape[2:4]), device="cuda")
            outs = {}
            for e in active:
                outs[e] = experts[e](image)[0]
                with torch.no_grad():
                    prediction[e] = outs[e]
            prediction.requires_grad_()
            (sx, sy), (f, ppx, ppy) = out["shifts"][0].tolist(), out["cameras"][0].tolist()
            loss = esac_loss(prediction, log_p, e_hyps[0], out["gt_poses"][0], opt.weightrot, opt.weighttrans,
                             opt.losscut, sx, sy, f, ppx, ppy, opt.threshold, opt.inlieralpha, opt.inlierbeta,
                             opt.maxreprojection, OUTPUT_SUBSAMPLE, expert_selection=opt.expertselection)
            loss.backward()
            for e in active:
                torch.autograd.backward(outs[e], prediction.grad[e])
                expert_opts[e].step()
                expert_opts[e].zero_grad(set_to_none=True)
            gating_opt.step()
            gating_opt.zero_grad(set_to_none=True)
            lines.append(train.log_line(it, float(loss.detach())).rstrip("\n"))
            it += 1
            if it % 250 == 0:
                print(f"eager twin: {it} iterations", flush=True)
    return [gating.state_dict()] + [m.state_dict() for m in experts], lines


def assert_same_model(path: Path, want):
    got = torch.load(path, map_location="cuda")
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert list(g) == list(w)
        for k in w:
            assert torch.equal(g[k], w[k]), k


def read_lines(path: Path):
    return path.read_text().splitlines()


def check_run(cwd: Path, argv, model: str, log: str):
    out = run(cwd, "esac_b200.train", *argv)
    assert "Done without errors." in out and "Epoch 0: mean loss" in out
    want, lines = twin(cwd, argv)
    assert_same_model(cwd / model, want)
    assert read_lines(cwd / log) == lines
    return want


def test_room_environment(tmp_path):
    write_environment(tmp_path, 3, [(48, 64), (64, 48)], seed=1)
    write_networks(tmp_path, 3, 1, "syn", seed=10)
    argv = ["-sid", "syn", "-hyps", "64", "-iter", "10", "-lr", "1e-4", "--seed", "4"]
    want = check_run(tmp_path, argv, "esac_syn.net", "log_esac_syn.txt")
    lines = read_lines(tmp_path / "log_esac_syn.txt")
    assert len(lines) == 1000 and lines[0].startswith("0 ") and lines[-1].startswith("999 ")
    start = torch.load(tmp_path / "expert_e0_syn.net")
    assert not torch.equal(want[1]["conv1.weight"].cpu(), start["conv1.weight"])    # the experts trained

    # the written model loads strictly into the library's modules and its device inference paths, and localize runs on it
    sds = torch.load(tmp_path / "esac_syn.net", map_location="cpu")
    Gating(3, 1).load_state_dict(sds[0], strict=True)
    GO.make_gating_class()(3, 1).load_state_dict(sds[0], strict=True)
    for sd in sds[1:]:
        Expert(torch.zeros(3)).load_state_dict(sd, strict=True)
    GatingNet(sds[0], "cuda")
    ExpertStack(sds[1:], "cuda")
    out = run(tmp_path, "esac_b200.localize", "-sid", "syn", "-hyps", "64")
    assert "Done without errors." in out and (tmp_path / "results_esac_syn.txt").exists()


def test_room_environment_expert_selection_refined(tmp_path):
    write_environment(tmp_path, 3, [(48, 64), (64, 48)], seed=2)
    write_networks(tmp_path, 3, 1, "syn", seed=20)
    for e in range(3):          # -ref reads the refined experts only: the plain files would be refused
        torch.save({}, tmp_path / f"expert_e{e}_syn.net")
    argv = ["-sid", "syn", "-hyps", "64", "-es", "-ref", "-lr", "1e-4", "-iter", "1"]
    check_run(tmp_path, argv, "es_syn.net", "log_es_syn.txt")
    assert not (tmp_path / "esac_syn.net").exists()


def test_room_environment_max_experts(tmp_path):
    write_environment(tmp_path, 3, [(48, 64), (64, 48)], seed=3)
    write_networks(tmp_path, 3, 1, "syn", seed=30)
    argv = ["-sid", "syn", "-hyps", "64", "-maxe", "1", "-iter", "1000", "-lr", "1e-4", "--seed", "11"]
    check_run(tmp_path, argv, "esac_syn.net", "log_esac_syn.txt")

    # in the captured loop itself: an expert without hypotheses keeps its parameters and Adam state, bitwise
    opt = train.options(argv)
    ds, draws, gating, experts, gating_opt, expert_opts = environment(tmp_path, opt)
    deterministic()
    loop = train.CapturedTrainLoop(opt, ds, gating, experts, gating_opt, expert_opts, len(draws))
    plan = train.epoch_plan(ds, draws)
    ds.load_plan(plan)

    def state(e):
        ts = [p.detach().clone() for p in experts[e].parameters()]
        return ts + [t.clone() for st in expert_opts[e].state.values() for t in (st["step"], st["exp_avg"], st["exp_avg_sq"])]
    idle_seen = 0
    for g in plan.groups[:24]:
        before = [state(e) for e in range(len(experts))]
        loop.graphs[g].replay()
        counts = loop.hist.tolist()
        assert sum(c > 0 for c in counts) == 1
        for e, c in enumerate(counts):
            same = all(torch.equal(a, b) for a, b in zip(before[e], state(e)))
            assert same == (c == 0), (e, counts)
            idle_seen += c == 0
    assert idle_seen == 48
    losses, statuses = loop.record(0, 24)
    assert np.isfinite(losses).all() and not statuses.any()


def test_clustered_environment(tmp_path):
    write_environment(tmp_path, 1, [(48, 64), (64, 48), (48, 64), (64, 48), (48, 64)], seed=4)
    write_networks(tmp_path, 2, 2, "cl", seed=40)
    argv = ["-c", "2", "-sid", "cl", "-hyps", "64", "-iter", "12", "-lr", "1e-4", "--seed", "2"]
    out = run(tmp_path, "esac_b200.train", *argv)
    assert "3 epoch(s) of 5 iterations" in out and "Epoch 2: mean loss" in out
    want, lines = twin(tmp_path, argv)
    assert_same_model(tmp_path / "esac_cl.net", want)
    assert read_lines(tmp_path / "log_esac_cl.txt") == lines and len(lines) == 15
    sds = torch.load(tmp_path / "esac_cl.net", map_location="cpu")
    assert GatingNet(sds[0], "cuda").capacity == 2


def test_gated_example_still_checks():
    r = subprocess.run([sys.executable, str(ROOT / "examples" / "train_step_gated_graph_synthetic.py"), "--images", "4",
                        "--experts", "4", "--maxexperts", "2", "--check"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("bitwise equal") == 4
