"""test_esac.py (code/test_esac.py) on the device, in one command:

    python -m esac_b200.localize -sid scene            # esac_scene.net, results_esac_scene.txt, poses_esac_scene.txt
    python -m esac_b200.localize -c 10 -sid aachen     # a clustered environment of 10 experts (gating capacity 2)

It takes test_esac.py's options with the same names and defaults, loads the model as expert_ensemble.py does (the ensemble
file, or with --testinit / --testrefined the individual gating_ and expert_e<i>_ files), builds the test set from the
folders of env_list.txt (esac_b200.data.from_room_folders, or from_cluster_folder with -c) and runs the reference's loop
as one CUDA graph per image shape: the image set's data step, GatingNet, the hypothesis draw, ExpertStack, the ESAC
forward and PoseEvaluator.update.  Every image is one replay; the host reads nothing back until the last replay, then
prints the reference's table and writes the results and pose files into the working directory.

Departures from test_esac.py:
  - the per-image console lines are not printed;
  - the draws use this library's counter-based generator (image i of a run draws with seed --seed + i, and the ESAC
    forward's sampling follows esac_b200.api.set_seed(--seed)), not torch.multinomial's stream;
  - the numerics are TF32 throughout (the reference's convolutions under torch's default cudnn.allow_tf32 = True).
"""
from __future__ import annotations

import argparse
import sys
import time

DEPARTURES = """departures from test_esac.py: the per-image console lines are not printed; the draws use this library's
counter-based generator (image i draws with seed --seed + i), not torch.multinomial's stream; the numerics are TF32
throughout."""


def options(argv=None):
    """test_esac.py's options (test_esac.py:15-59), with the same names and defaults, and --seed."""
    p = argparse.ArgumentParser(description="Test ESAC on the device.", epilog=DEPARTURES,
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--model", "-m", default="",
                   help="ensemble model file, if empty we use the default file name + the session ID")
    p.add_argument("--testinit", "-tinit", action="store_true",
                   help="load individual expert networks and gating, used for testing before end-to-end training, we use "
                        "the default file names + session ID")
    p.add_argument("--testrefined", "-tref", action="store_true",
                   help="load individual refined expert networks and gating, used for testing before end-to-end training, "
                        "we use the default file names + session ID + refined post fix")
    p.add_argument("--hypotheses", "-hyps", type=int, default=256, help="number of hypotheses, i.e. number of RANSAC iterations")
    p.add_argument("--threshold", "-t", type=float, default=10, help="inlier threshold in pixels")
    p.add_argument("--inlieralpha", "-ia", type=float, default=100,
                   help="alpha parameter of the soft inlier count; Controls the softness of the hypotheses score "
                        "distribution; lower means softer")
    p.add_argument("--inlierbeta", "-ib", type=float, default=0.5,
                   help="beta parameter of the soft inlier count; controls the softness of the sigmoid; lower means softer")
    p.add_argument("--maxreprojection", "-maxr", type=float, default=100,
                   help="maximum reprojection error; reprojection error is clamped to this value for stability")
    p.add_argument("--rotthreshold", "-rt", type=float, default=5, help="acceptance threshold of rotation error in degree")
    p.add_argument("--transthreshold", "-tt", type=float, default=5,
                   help="acceptance threshold of translation error in centimeters")
    p.add_argument("--expertselection", "-es", action="store_true", help="select one expert instead of distributing hypotheses")
    p.add_argument("--oracleselection", "-os", action="store_true", help="always select the ground truth expert")
    p.add_argument("--clusters", "-c", type=int, default=-1,
                   help="number of clusters the environment should be split into, corresponds to the number of desired "
                        "experts")
    p.add_argument("--session", "-sid", default="",
                   help="custom session name appended to output files, useful to separate different runs of a script")
    p.add_argument("--seed", type=int, default=0,
                   help="seed of the hypothesis draws (image i draws with seed + i) and of the ESAC forward's sampling")
    opt = p.parse_args(argv)
    if opt.oracleselection and opt.clusters >= 0:
        p.error("--oracleselection needs the ground-truth expert of each image; a clustered environment (-c) has none")
    return opt


def model_files(opt, num_experts: int):
    """The files expert_ensemble.py loads (:94-112) for test_esac.py's options (:88-102): ("ensemble", path) or
    ("individual", gating path, [expert paths])."""
    if opt.testrefined or opt.testinit:
        session = opt.session + ("_refined" if opt.testrefined else "")
        return ("individual", "./gating_%s.net" % opt.session,
                ["./expert_e%d_%s.net" % (i, session) for i in range(num_experts)])
    if opt.model:
        return ("ensemble", opt.model)
    return ("ensemble", ("es_%s.net" if opt.expertselection else "esac_%s.net") % opt.session)


def output_session(opt) -> str:
    """The session name of the output files, with test_esac.py's prefixes (:104-114)."""
    session = opt.session
    if opt.testinit:
        session = "init_" + session
    if opt.testrefined:
        session = "ref_" + session
    if opt.expertselection:
        session = "es_" + session
    if opt.oracleselection:
        session = "os_" + session
    return session


def load_model(opt, num_experts: int):
    """(gating state dict, [expert state dicts]) from the files model_files names."""
    import torch
    files = model_files(opt, num_experts)
    if files[0] == "individual":
        return torch.load(files[1], map_location="cpu"), [torch.load(f, map_location="cpu") for f in files[2]]
    sds = torch.load(files[1], map_location="cpu")
    if len(sds) != num_experts + 1:
        raise RuntimeError(f"{files[1]} holds {len(sds) - 1} experts; the environment has {num_experts}")
    return sds[0], list(sds[1:])


def rgb_files(clustered: bool, env_list: str = "env_list.txt") -> list:
    """The test set's rgb files in the image set's order (each scene's sorted test/rgb/, scenes in env_list order)."""
    from .data import _listed
    with open(env_list, "r") as f:
        scenes = [line.split()[0] for line in f.readlines() if line.split()]
    if clustered:
        scenes = scenes[:1]
    return [f for s in scenes for f in _listed(s + "/test/rgb/")]


def strip_file_name(f: str) -> str:
    """util.strip_file_name: the file name without its path and the Aachen prefixes."""
    f = f.split("/")[-1]
    for ign in ("db_", "query_day_milestone_", "query_day_nexus4_", "query_day_nexus5x_", "query_night_nexus5x_"):
        if f.startswith(ign):
            f = f[len(ign):]
    return f


class CapturedTestLoop:
    """The test step of every shape group of `dataset`, captured once each: data step, gating, draw, experts, forward,
    evaluation.  Workspaces are reserved for the largest group before the first capture and shared by the graphs."""

    def __init__(self, opt, dataset, gating, stack, clustered: bool):
        import torch

        from . import api
        from .compat import OUTPUT_SUBSAMPLE
        from .data import ClusterDraws, Plan, RoomDraws, cluster_jitter
        from .evaluate import PoseEvaluator
        from .experts import prediction_size
        self.opt, self.dataset = opt, dataset
        E, M = gating.E, opt.hypotheses
        dev = dataset.device
        draws = ClusterDraws(len(dataset), jitter=cluster_jitter(False)) if clustered else \
            RoomDraws(dataset.scene_counts, training=False)
        self.plan = dataset.plan(draws, batch=1, shuffle=False, shift=False)
        self.evaluator = PoseEvaluator(E, len(dataset), device=dev, clustered=clustered)
        thresholds = (opt.threshold, opt.inlieralpha, opt.inlierbeta, opt.maxreprojection, OUTPUT_SUBSAMPLE)
        self.seed = torch.tensor([opt.seed], dtype=torch.int64, device=dev)
        log_p, probs = torch.zeros(1, E, device=dev), torch.zeros(1, E, device=dev)
        e_hyps = torch.zeros(1, M, dtype=torch.int64, device=dev)
        hist = torch.zeros(1, E, device=dev)
        draw_status = torch.zeros(1, dtype=torch.int32, device=dev)
        pose = torch.zeros(1, 4, 4, device=dev)
        expert = torch.zeros(1, dtype=torch.int64, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)

        groups = sorted(set(self.plan.groups))
        shapes = [dataset.groups[g][:2] for g in groups]
        for h_, w_ in shapes:          # every workspace at its largest before the first capture
            gating.reserve(1, h_, w_)
            stack.reserve(1, h_, w_)
        api.reserve_forward_async(1, E, max(prediction_size(*s)[0] for s in shapes),
                                  max(prediction_size(*s)[1] for s in shapes), M, OUTPUT_SUBSAMPLE)

        def step(g, prediction):
            with torch.no_grad():
                out = dataset.step(g)
                image = out["image"]
                gating.forward_async(image, log_p, probs)
                if opt.oracleselection:                            # test_esac.py:166-168
                    probs.zero_()
                    probs.scatter_(1, out["scenes"].view(1, 1), 1.0)
                api.assign_hypotheses_async(probs, M, self.seed, e_hyps, hist, draw_status,
                                            expertSelection=opt.expertselection or opt.oracleselection)
                self.seed.add_(1)
                stack.forward_async(image, hist, prediction)
            api.forward_async(prediction, e_hyps, out["shifts"], out["cameras"], *thresholds, pose, expert, status)
            self.evaluator.update(pose, out["gt_poses"], expert, out["scenes"], hist=hist, status=status)

        self.graphs = {}
        self.keep = [log_p, probs, e_hyps, hist, draw_status, pose, expert, status, step]
        for g in groups:
            Hg, Wg = dataset.groups[g][:2]
            prediction = torch.zeros((1, E, 3) + prediction_size(Hg, Wg), device=dev)
            first = self.plan.groups.index(g)      # the warm-up runs on the group's first image
            dataset.load_plan(Plan(self.plan.rows[first:first + 1], [g], 1))
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                step(g, prediction)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step(g, prediction)
            self.graphs[g] = graph
            self.keep.append(prediction)

    def run(self) -> float:
        """Replays every step of the plan in order; returns the host seconds around the replays."""
        import torch

        from . import api
        self.dataset.load_plan(self.plan)
        self.evaluator.reset()
        self.seed.fill_(self.opt.seed)
        api.set_seed(self.opt.seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for g in self.plan.groups:
            self.graphs[g].replay()
        torch.cuda.synchronize()
        return time.perf_counter() - t0


def main(argv=None) -> int:
    opt = options(argv)
    from .data import from_cluster_folder, from_room_folders
    from .experts import ExpertStack
    from .gating_net import GatingNet
    clustered = opt.clusters >= 0
    if clustered:
        dataset = from_cluster_folder("test", training=False)
        num_experts, capacity = opt.clusters, 2     # test_esac.py:70-78
    else:
        dataset = from_room_folders("test", training=False)
        num_experts, capacity = len(dataset.scene_counts), 1
    gating_sd, expert_sds = load_model(opt, num_experts)
    dev = dataset.device
    gating = GatingNet(gating_sd, dev)
    if (gating.E, gating.capacity) != (num_experts, capacity):
        raise RuntimeError(f"the gating network has {gating.E} experts at capacity {gating.capacity}; the environment "
                           f"needs {num_experts} at capacity {capacity}")
    stack = ExpertStack(expert_sds, dev)
    session = output_session(opt)
    names = [strip_file_name(f) for f in rgb_files(clustered)]
    if len(names) != len(dataset):
        raise RuntimeError(f"{len(names)} test files listed for a set of {len(dataset)} images")

    print("Environment has", len(dataset), "test images.")
    loop = CapturedTestLoop(opt, dataset, gating, stack, clustered)
    seconds = loop.run()
    table = loop.evaluator.table(opt.rotthreshold, opt.transthreshold, average=not clustered)
    with open("results_esac_%s.txt" % session, "w") as f:
        f.write("".join(line + "\n" for line in table["results"]))
    with open("poses_esac_%s.txt" % session, "w") as f:
        f.write("".join(line + "\n" for line in loop.evaluator.pose_lines(names)))
    print("\n".join(table["console"]))
    print("\n" + table["experts"][0])
    print(table["experts"][1])
    if table["excluded"]:
        print(f"{table['excluded']} image(s) left out of the table: forward status != 0")
    print("\nAvg. Time: %.3fs" % (seconds / len(dataset)))
    print("\nDone without errors.")
    return 0


if __name__ == "__main__":
    sys.exit(main())
