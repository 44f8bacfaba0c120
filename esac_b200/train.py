"""train_esac.py (code/train_esac.py) on the device, in one command:

    python -m esac_b200.train -sid scene               # gating_scene.net + expert_e<i>_scene.net -> esac_scene.net
    python -m esac_b200.train -c 10 -sid aachen -ref   # a clustered environment of 10 experts, from the refined experts

It takes train_esac.py's options with the same names and defaults, loads the networks as ExpertEnsemble.load_experts does
(gating_<sid>.net and expert_e<i>_<sid>.net, or expert_e<i>_<sid>_refined.net with -ref), builds the training set from the
folders of env_list.txt (esac_b200.data.from_room_folders, or from_cluster_folder with -c and the training colour jitter)
and runs the reference's end-to-end training loop as one CUDA graph per image shape.  A step is the image set's data step
(image, jitter, normalisation, random shift, camera and pose), the gating network and exp, the hypothesis draw with
util.clamp_probs, the experts that drew hypotheses (gate.ExpertGate: the others are neither run nor stepped), the ESAC
loss with the gating gradient (autograd.esac_loss_async), each active expert's backward and Adam step, and the gating
network's Adam step.  The networks (networks.Expert, networks.Gating) and their optimisers are torch; the step is
captured as it is.  The loss and the statuses of every iteration are kept in device memory and read back once per epoch.

As train_esac.py does, it runs ceil(-iter / epoch length) whole epochs, each on a fresh shuffled draw of the training set
(a room environment's epoch is 1000 random images, a clustered one's is its image count), saves the model as
ExpertEnsemble.save does ([gating, expert_0, ...]) to esac_<sid>.net (es_<sid>.net with -es) at the start of every epoch,
and writes the log log_esac_<sid>.txt (log_es_<sid>.txt) in its line format, '%d %f \\n'.  If an iteration's hypothesis
draw or ESAC backward reports a failure (a NaN gating output, say), the command stops before the next save, names the
first such iteration, and exits with status 1.

--seed seeds everything random: random.seed and torch.manual_seed before the first epoch's draw of the training set (the
shuffles, the scene and image choices, the jitter and the shifts, in the reference's order; esac_b200.data.make_plan),
the hypothesis draws (iteration i draws with seed --seed + i) and the ESAC backward's sampling (esac_b200.api.set_seed).

Departures from train_esac.py:
  - no console line per iteration: one line per epoch, with the epoch's mean loss and seconds;
  - the draws use this library's counter-based generator, not torch.multinomial's stream;
  - the convolutions are TF32 under torch's defaults, with cuDNN's deterministic algorithms, so that a run is
    reproducible from --seed;
  - the log holds each loss as the float32 the ESAC loss node returns;
  - the model is saved once more after the last iteration.
"""
from __future__ import annotations

import argparse
import math
import random
import sys
import time

DEPARTURES = """departures from train_esac.py: no console line per iteration, one line per epoch (mean loss, seconds); the
draws use this library's counter-based generator (iteration i draws with seed --seed + i), not torch.multinomial's stream;
the convolutions are TF32 under torch's defaults, with cuDNN's deterministic algorithms; the log holds each loss as a
float32; the model is saved once more after the last iteration."""


def options(argv=None):
    """train_esac.py's options (train_esac.py:20-63), with the same names and defaults, and --seed."""
    p = argparse.ArgumentParser(description="Train an ensemble of experts end-to-end, minimizing the final pose error, on "
                                            "the device.", epilog=DEPARTURES,
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--hypotheses", "-hyps", type=int, default=256, help="hypotheses per image (RANSAC iterations)")
    p.add_argument("--threshold", "-t", type=float, default=10, help="inlier threshold, in pixels")
    p.add_argument("--inlieralpha", "-ia", type=float, default=100,
                   help="alpha of the soft inlier count: the softness of the hypothesis score distribution (lower is "
                        "softer)")
    p.add_argument("--inlierbeta", "-ib", type=float, default=0.5,
                   help="beta of the soft inlier count: the softness of its sigmoid (lower is softer)")
    p.add_argument("--maxreprojection", "-maxr", type=float, default=100,
                   help="reprojection errors are clamped to this value, for stability")
    p.add_argument("--learningrate", "-lr", type=float, default=0.000001, help="learning rate of every network")
    p.add_argument("--iterations", "-iter", type=int, default=50000,
                   help="training iterations (model updates); whole epochs are run until they reach it")
    p.add_argument("--weightrot", "-wr", type=float, default=1.0, help="weight of the rotation error (degrees)")
    p.add_argument("--weighttrans", "-wt", type=float, default=100.0, help="weight of the translation error (metres)")
    p.add_argument("--losscut", "-lc", type=float, default=100.0,
                   help="the pose loss grows as a square root above this value")
    p.add_argument("--clusters", "-c", type=int, default=-1,
                   help="train on a clustered environment of this many experts (gating capacity 2); -1: a room "
                        "environment, one expert per scene of env_list.txt")
    p.add_argument("--maxexperts", "-maxe", type=int, default=-1,
                   help="draw hypotheses from at most this many of the most likely experts per image; -1: no limit")
    p.add_argument("--expertselection", "-es", action="store_true",
                   help="draw one expert per image instead of distributing the hypotheses")
    p.add_argument("--session", "-sid", default="", help="session name in the input and output file names")
    p.add_argument("--refined", "-ref", action="store_true",
                   help="start from the refined experts (expert_e<i>_<sid>_refined.net)")
    p.add_argument("--seed", type=int, default=0,
                   help="seed of the training set's draws, of the hypothesis draws (iteration i draws with seed + i) and "
                        "of the ESAC backward's sampling")
    opt = p.parse_args(argv)
    if opt.iterations < 1 or opt.hypotheses < 1:
        p.error("-iter and -hyps must be positive")
    return opt


def _individual(opt) -> argparse.Namespace:
    """The options under which localize's helpers name and load the individual files of load_experts."""
    return argparse.Namespace(testinit=not opt.refined, testrefined=opt.refined, session=opt.session, model="",
                              expertselection=False)


def input_files(opt, num_experts: int) -> tuple:
    """(gating file, [expert files]) that ExpertEnsemble.load_experts(session, ref) reads (expert_ensemble.py:94-103)."""
    from .localize import model_files
    _, gating, experts = model_files(_individual(opt), num_experts)
    return gating, experts


def output_files(opt) -> tuple:
    """(model file, log file) of train_esac.py:87-92."""
    prefix = "es" if opt.expertselection else "esac"
    return "%s_%s.net" % (prefix, opt.session), "log_%s_%s.txt" % (prefix, opt.session)


def epochs(iterations: int, epoch_length: int) -> int:
    """train_esac.py:96: whole epochs of the training set's draws (len(trainset)) that reach `iterations`."""
    return math.ceil(iterations / epoch_length)


def log_line(iteration: int, loss: float) -> str:
    """One line of the training log (train_esac.py:186)."""
    return "%d %f \n" % (iteration, loss)


def training_draws(dataset, clustered: bool):
    """The random calls of the reference's training set: RoomDataset("training", training=True) (an epoch of 1000 random
    images), or ClusterDataset("training", training=True) with its training colour jitter."""
    from .data import ClusterDraws, RoomDraws, cluster_jitter
    if clustered:
        return ClusterDraws(len(dataset), jitter=cluster_jitter(True))
    return RoomDraws(dataset.scene_counts, training=True)


def epoch_plan(dataset, draws):
    """One epoch of the reference loop's DataLoader(trainset, shuffle=True) and util.random_shift, as steps of one image."""
    return dataset.plan(draws, batch=1, shuffle=True, shift=True)


def load_networks(opt, num_experts: int, capacity: int, device):
    """(networks.Gating, [networks.Expert]) on `device`, loaded from input_files.  A file whose network has the wrong number
    of experts, the wrong capacity, or a missing, extra or misshapen key is refused by name."""
    import torch

    from . import experts as X
    from . import gating_net as G
    from .networks import Expert, Gating
    gating_file, expert_files = input_files(opt, num_experts)
    gating_sd = torch.load(gating_file, map_location="cpu")
    try:
        E, c = G.network_size(gating_sd)
    except RuntimeError as e:
        raise RuntimeError(f"{gating_file}: {e}") from None
    if (E, c) != (num_experts, capacity):
        raise RuntimeError(f"{gating_file}: the gating network has {E} experts at capacity {c}; the environment needs "
                           f"{num_experts} at capacity {capacity}")
    X._check_state_dict(gating_file, gating_sd, G.state_dict_shapes(E, c), "Gating")
    expert_sds = [torch.load(f, map_location="cpu") for f in expert_files]
    for f, sd in zip(expert_files, expert_sds):
        X._check_state_dict(f, sd, X.state_dict_shapes(), "Expert")
    gating = Gating(E, c).to(device)
    gating.load_state_dict(gating_sd)
    nets = []
    for sd in expert_sds:
        nets.append(Expert(sd["mean"]).to(device))
        nets[-1].load_state_dict(sd)
    return gating, nets


def optimizers(opt, gating, experts) -> tuple:
    """One Adam for the gating network and one per expert (expert_ensemble.py:19-37), capturable, their state created."""
    import torch

    from .networks import init_adam_state
    gating_opt = torch.optim.Adam(gating.parameters(), lr=opt.learningrate, capturable=True)
    expert_opts = [torch.optim.Adam(m.parameters(), lr=opt.learningrate, capturable=True) for m in experts]
    for o in [gating_opt] + expert_opts:
        init_adam_state(o)
    return gating_opt, expert_opts


def save_model(path: str, gating, experts):
    """ExpertEnsemble.save (expert_ensemble.py:84-92): [gating state dict, expert state dicts...]."""
    import torch
    torch.save([gating.state_dict()] + [m.state_dict() for m in experts], path)


class CapturedTrainLoop:
    """The training step of every shape group of `dataset`, captured once each (train_esac.py:105-183): data step, gating,
    draw, the experts that drew hypotheses, ESAC loss and backward, the active experts' and the gating network's Adam
    steps, and the iteration's record.  The graphs share the networks, the optimisers' state and the buffers; the
    workspaces are reserved for the largest group before the first capture.  Warming up and capturing leave the networks
    and the optimisers as they were.  `iterations`: the record's length (every iteration of the run)."""

    def __init__(self, opt, dataset, gating, experts, gating_opt, expert_opts, iterations: int):
        import numpy as np
        import torch

        from . import api
        from .autograd import esac_loss_async
        from .compat import OUTPUT_SUBSAMPLE
        from .data import Plan
        from .experts import prediction_size
        from .gate import ExpertGate
        self.opt, self.dataset = opt, dataset
        E, M = len(experts), opt.hypotheses
        dev = dataset.device
        self.seed = torch.tensor([opt.seed], dtype=torch.int64, device=dev)
        self.iteration = torch.zeros(1, dtype=torch.int64, device=dev)
        self.losses = torch.zeros(iterations, device=dev)
        self.statuses = torch.zeros((iterations, 2), dtype=torch.int32, device=dev)   # draw, ESAC backward
        e_hyps = torch.zeros(M, dtype=torch.int64, device=dev)
        self.hist = hist = torch.zeros(E, device=dev)        # the last replay's hypothesis histogram
        draw_status = torch.zeros((), dtype=torch.int32, device=dev)
        status = torch.zeros((), dtype=torch.int32, device=dev)
        params = (opt.weightrot, opt.weighttrans, opt.losscut, opt.threshold, opt.inlieralpha, opt.inlierbeta,
                  opt.maxreprojection, OUTPUT_SUBSAMPLE)

        def step(g, gate, prediction):
            out = dataset.step(g)                                                               # train_esac.py:105-125
            image = out["image"]
            gating_log_probs = gating(image)                                                    # :128
            gating_probs = torch.exp(gating_log_probs).detach()[0]
            api.assign_hypotheses_async(gating_probs, M, self.seed, e_hyps, hist, draw_status,  # :131-141
                                        maxExperts=opt.maxexperts, expertSelection=opt.expertselection)
            self.seed.add_(1)
            gate.arm(hist)
            outs = [None] * E
            with torch.no_grad():
                prediction.zero_()

            def forward(e):                                                                     # :143-145
                outs[e] = experts[e](image)[0]
                with torch.no_grad():
                    prediction[e].copy_(outs[e])
            for e in range(E):
                gate.run(e, lambda e=e: forward(e))
            leaf = prediction.detach().requires_grad_()
            loss = esac_loss_async(leaf, gating_log_probs, e_hyps, out["gt_poses"][0], out["shifts"][0],   # :151-176
                                   out["cameras"][0], *params, expert_selection=opt.expertselection, status=status)
            loss.backward()                                                                     # :178-180

            def backward(e):                                                                    # ensemble.update
                torch.autograd.backward(outs[e], leaf.grad[e])
                expert_opts[e].step()
                expert_opts[e].zero_grad(set_to_none=True)
            for e in range(E):
                gate.run(e, lambda e=e: backward(e))
            gating_opt.step()
            gating_opt.zero_grad(set_to_none=True)
            with torch.no_grad():                                                               # :185-186
                self.losses.index_copy_(0, self.iteration, loss.detach().view(1))
                self.statuses.index_copy_(0, self.iteration, torch.stack((draw_status, status)).view(1, 2))
                self.iteration.add_(1)

        groups = list(range(len(dataset.groups)))
        shapes = [prediction_size(*dataset.groups[g][:2]) for g in groups]
        api.reserve_backward_async(1, E, max(s[0] for s in shapes), max(s[1] for s in shapes), M, OUTPUT_SUBSAMPLE)
        state = [p for m in [gating] + list(experts) for p in m.parameters()]
        state += [t for o in [gating_opt] + list(expert_opts) for st in o.state.values()
                  for t in (st["step"], st["exp_avg"], st["exp_avg_sq"])]
        with torch.no_grad():
            before = [t.detach().clone() for t in state]
        self.graphs, self.keep = {}, [e_hyps, hist, draw_status, status, step]
        for g, (h, w) in zip(groups, shapes):
            gate = ExpertGate(E, dev)
            prediction = torch.zeros((E, 3, h, w), device=dev)
            row = np.zeros(1, api.DATA_ROW)                    # the group's first image, unshifted, unjittered
            row["image"] = int(np.flatnonzero(dataset.group_of == g)[0])
            side = torch.cuda.Stream(dev)
            for _ in range(3):                                 # torch's lazy initialisations, off the capture
                dataset.load_plan(Plan(row, [g], 1))
                self.iteration.zero_()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    step(g, gate, prediction)
                torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph(keep_graph=True)
            with torch.cuda.graph(graph):
                step(g, gate, prediction)
            gate.finalize(graph)
            self.graphs[g] = graph
            self.keep += [gate, prediction]
        with torch.no_grad():
            for t, b in zip(state, before):
                t.copy_(b)
        self.seed.fill_(opt.seed)
        self.iteration.zero_()
        api.set_seed(opt.seed)
        torch.cuda.synchronize(dev)

    def run(self, plan) -> float:
        """Replays the steps of one epoch's plan in order; returns the host seconds around the replays."""
        import torch
        self.dataset.load_plan(plan)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for g in plan.groups:
            self.graphs[g].replay()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def record(self, begin: int, end: int) -> tuple:
        """The losses (float32) and the (draw, backward) statuses of iterations [begin, end), read back in one copy each."""
        return self.losses[begin:end].cpu().numpy(), self.statuses[begin:end].cpu().numpy()


def main(argv=None) -> int:
    opt = options(argv)
    import torch

    from .data import from_cluster_folder, from_room_folders
    clustered = opt.clusters >= 0
    if clustered:                                          # train_esac.py:67-81
        dataset = from_cluster_folder("training", training=True)
        num_experts, capacity = opt.clusters, 2
    else:
        dataset = from_room_folders("training", training=True)
        num_experts, capacity = len(dataset.scene_counts), 1
    draws = training_draws(dataset, clustered)
    gating, experts = load_networks(opt, num_experts, capacity, dataset.device)
    gating_opt, expert_opts = optimizers(opt, gating, experts)
    model_file, log_file = output_files(opt)
    n_epochs = epochs(opt.iterations, len(draws))
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False

    print("Environment has", len(dataset), "training images;", n_epochs, "epoch(s) of", len(draws), "iterations.")
    loop = CapturedTrainLoop(opt, dataset, gating, experts, gating_opt, expert_opts, n_epochs * len(draws))
    random.seed(opt.seed)
    torch.manual_seed(opt.seed)
    with open(log_file, "w", 1) as log:
        def close_epoch(epoch: int, seconds: float) -> bool:
            begin, end = epoch * len(draws), (epoch + 1) * len(draws)
            losses, statuses = loop.record(begin, end)
            bad = [i for i in range(end - begin) if statuses[i].any()]
            good = bad[0] if bad else end - begin
            log.write("".join(log_line(begin + i, float(losses[i])) for i in range(good)))
            if bad:
                i = bad[0]
                print(f"iteration {begin + i}: draw status {int(statuses[i, 0])}, ESAC backward status "
                      f"{int(statuses[i, 1])}; stopped before saving {model_file}", file=sys.stderr)
                return False
            print("Epoch %d: mean loss %.2f, %.2fs" % (epoch, float(losses.mean()), seconds), flush=True)
            return True

        for epoch in range(n_epochs):
            print("=== Epoch: %d ======================================" % epoch)
            if epoch and not close_epoch(epoch - 1, seconds):
                return 1
            save_model(model_file, gating, experts)
            print("Saved model.")
            seconds = loop.run(epoch_plan(dataset, draws))
        if not close_epoch(n_epochs - 1, seconds):
            return 1
        save_model(model_file, gating, experts)
        print("Saved model.")
    print("Done without errors.")
    return 0


if __name__ == "__main__":
    sys.exit(main())
