"""Eager esac.backward against the stream-ordered backward, uncaptured and as CUDA-graph replays, and a whole training step
eager against its captured form (GPU only).

For every shape, R images end in ONE torch.cuda.synchronize():
  eager   esac.backward on CUDA tensors (it synchronises inside every call),
  async   api.backward_async in a loop, uncaptured,
  graph   replays of one captured api.backward_async,
  step    a training step of examples/train_step_graph_synthetic.py's stand-ins (gating, torch.multinomial, every expert,
          the ESAC loss, loss.backward(), Adam): eager with esac_loss, against replays of the step captured with
          esac_loss_async and Adam(capturable=True).
Reported per image: host wall time over the R images, and device time between CUDA events around them.  The shapes are
those of tools/forward_async_timing.py.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/backward_async_timing.py [--images 50] [--json out.json]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "examples"))
import torch  # noqa: E402

import esac_b200.api as api  # noqa: E402
from esac_b200.autograd import esac_loss, esac_loss_async  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402
from train_step_synthetic import TinyExpert, TinyGating  # noqa: E402

SHAPES = [("60x80 sub 8, E=1 M=64", dict(E=1, H=60, W=80, M=64, sub=8)),
          ("60x80 sub 8, E=7 M=256", dict(E=7, H=60, W=80, M=256, sub=8)),
          ("60x80 sub 8, E=19 M=256", dict(E=19, H=60, W=80, M=256, sub=8)),
          ("60x80 sub 8, E=20 M=1024", dict(E=20, H=60, W=80, M=1024, sub=8)),
          ("480x640 sub 1, E=7 M=256", dict(E=7, H=480, W=640, M=256, sub=1))]
LOSS = (1.0, 100.0, 100.0)
TAIL = (10.0, 100.0, 0.5, 100.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, R):
    """(host ms per image, device ms per image) of R calls of fn ending in one synchronise."""
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(R):
        fn()
    b.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / R
    return wall, a.elapsed_time(b) / R


def capture(fn, reset=lambda: None):
    """fn captured after three warm-up runs on a side stream; reset() runs before each of them and before the capture."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            reset()
            fn()
    torch.cuda.current_stream().wait_stream(side)
    reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def training_steps(sc, E, M, sub):
    """(eager step, captured step's graph, what the graph reads) on the stand-ins, one image of the scene's size.  A graph
    holds no reference to the tensors it reads: the caller keeps the third element alive for as long as it replays."""
    image = torch.rand(1, 1, sc.coords.shape[2] * sub, sc.coords.shape[3] * sub, device="cuda")
    prior = torch.from_numpy(sc.coords).cuda()
    gt = torch.from_numpy(sc.gt_pose).cuda()
    shift = torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda")
    cam = torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda")

    def nets(capturable):
        torch.manual_seed(0)
        experts = [TinyExpert().cuda() for _ in range(E)]
        for e in range(E):
            experts[e].see(prior[e])
        gating = TinyGating(E).cuda()
        opts = [torch.optim.Adam(m.parameters(), lr=1e-5, capturable=capturable) for m in experts]
        return experts, gating, opts + [torch.optim.Adam(gating.parameters(), lr=1e-4, capturable=capturable)]

    experts, gating, opts = nets(False)

    def eager():
        glp = gating(image)
        e_hyps = torch.multinomial(torch.exp(glp).detach()[0], M, replacement=True)
        prediction = torch.stack([experts[e](image)[0] for e in range(E)])
        loss = esac_loss(prediction, glp, e_hyps, gt, *LOSS, *sc.params)
        for o in opts:
            o.zero_grad(set_to_none=True)
        loss.backward()
        for o in opts:
            o.step()

    g_experts, g_gating, g_opts = nets(True)

    def step():
        glp = g_gating(image)
        e_hyps = torch.multinomial(torch.exp(glp).detach()[0], M, replacement=True)
        prediction = torch.stack([g_experts[e](image)[0] for e in range(E)])
        loss = esac_loss_async(prediction, glp, e_hyps, gt, shift, cam, *LOSS, *TAIL, sub)
        loss.backward()
        for o in g_opts:
            o.step()

    def reset():   # the captured backward then allocates the gradients and sets them on every replay
        for o in g_opts:
            o.zero_grad(set_to_none=True)

    return eager, capture(step, reset), (step, image, gt, shift, cam, g_experts, g_gating, g_opts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", "-R", type=int, default=50)
    ap.add_argument("--json", help="also write the table here")
    opt = ap.parse_args()
    R = opt.images
    name = card()
    print(f"card (name, power limit, max SM clock): {name}", flush=True)
    rows = []
    for _, kw in SHAPES:   # every shape before the first capture: a captured workspace never grows
        api.reserve_backward_async(1, kw["E"], kw["H"], kw["W"], kw["M"], kw["sub"])
    for label, kw in SHAPES:
        sc = make_scene(seed=7, **kw)
        E, M, sub = kw["E"], kw["M"], kw["sub"]
        coords = torch.from_numpy(sc.coords).cuda()
        grads = torch.zeros_like(coords)
        assign = torch.from_numpy(sc.assign).cuda()
        gt = torch.from_numpy(sc.gt_pose).cuda()
        shifts = torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda")
        cams = torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda")
        loss = torch.zeros((), dtype=torch.float64, device="cuda")
        status = torch.zeros((), dtype=torch.int32, device="cuda")

        def eager():
            api.backward(coords, grads, assign, gt, *LOSS, *sc.params)

        def stream_ordered():
            api.backward_async(coords, grads, assign, gt, shifts, cams, *LOSS, *TAIL, sub, loss, status)

        for _ in range(3):
            eager()
            stream_ordered()
        torch.cuda.synchronize()
        st = api.last_stats()
        g = capture(stream_ordered)
        step_eager, step_graph, step_inputs = training_steps(sc, E, M, sub)
        res = {"shape": label, "kernel_launches": st["kernel_launches"], "n_contrib": st["n_contrib"],
               "refine_group": st["refine_group"]}
        for kind, fn in (("eager", eager), ("async", stream_ordered), ("graph", g.replay), ("step_eager", step_eager),
                         ("step_graph", step_graph.replay)):
            res[kind] = timed(fn, R)
        torch.cuda.synchronize()
        assert int(status) == 0
        rows.append(res)
        print(f"{label:26s} contributing {st['n_contrib']:4d} group {st['refine_group']:3d} | host ms/image: eager "
              f"{res['eager'][0]:7.3f} async {res['async'][0]:7.3f} graph {res['graph'][0]:7.3f} step eager "
              f"{res['step_eager'][0]:7.3f} step graph {res['step_graph'][0]:7.3f} | device ms/image: eager "
              f"{res['eager'][1]:7.3f} async {res['async'][1]:7.3f} graph {res['graph'][1]:7.3f} step eager "
              f"{res['step_eager'][1]:7.3f} step graph {res['step_graph'][1]:7.3f}", flush=True)
        del g, step_graph, step_inputs
    if opt.json:
        Path(opt.json).write_text(json.dumps({"card": name, "images": R, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
