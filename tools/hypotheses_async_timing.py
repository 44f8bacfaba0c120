"""The eager hypotheses node against the stream-ordered one, uncaptured and as CUDA-graph replays, and a custom-loss
training step eager against its captured form (GPU only).

For every shape, R images end in ONE torch.cuda.synchronize():
  eager   api.hypotheses_forward + api.hypotheses_backward on CUDA tensors (each synchronises inside),
  async   api.hypotheses_forward_async + api.hypotheses_backward_async in a loop, uncaptured,
  graph   replays of one captured forward + backward,
  step    the DSAC* step of examples/custom_loss_step_graph_synthetic.py (stand-in gating and experts, torch.multinomial,
          the node, the DSAC* loss, the REINFORCE gating term, backward(), Adam): eager on esac_hypotheses, against replays
          of the step captured on esac_hypotheses_async with Adam(capturable=True).
Reported per image: host wall time over the R images, and device time between CUDA events around them.  The shapes are
those of tools/backward_async_timing.py.  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/hypotheses_async_timing.py [--images 50] [--json out.json]
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "examples"))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import torch  # noqa: E402

import esac_b200.api as api  # noqa: E402
from backward_async_timing import SHAPES, TAIL, capture, card, timed  # noqa: E402
from custom_loss_step_graph_synthetic import FEATS, Nets, step  # noqa: E402
from esac_b200.autograd import esac_hypotheses, esac_hypotheses_async  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402


def training_steps(sc, E, M, sub):
    """(eager step, captured step's graph, what the graph reads) on the stand-ins; the caller keeps the third alive."""
    prior = torch.from_numpy(sc.coords).cuda()
    feats = torch.randn(1, FEATS, device="cuda")
    gt = torch.from_numpy(sc.gt_pose).cuda()
    shift = torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda")
    cam = torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda")

    def nets(capturable):
        torch.manual_seed(0)
        n = Nets(E, FEATS).cuda()
        return n, torch.optim.Adam(n.parameters(), lr=1e-4, capturable=capturable)

    e_nets, e_opt = nets(False)

    def eager():
        e_opt.zero_grad(set_to_none=True)
        step(e_nets, prior, feats, gt, lambda p, h: esac_hypotheses(p, h, *sc.params), M=M)
        e_opt.step()

    g_nets, g_opt = nets(True)

    def captured():
        step(g_nets, prior, feats, gt, lambda p, h: esac_hypotheses_async(p, h, shift, cam, *TAIL, sub), M=M)
        g_opt.step()

    return eager, capture(captured, lambda: g_opt.zero_grad(set_to_none=True)), (prior, feats, gt, shift, cam, g_nets, g_opt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", "-R", type=int, default=50)
    ap.add_argument("--json", help="also write the table here")
    opt = ap.parse_args()
    R = opt.images
    name = card()
    print(f"card (name, power limit, max SM clock): {name}", flush=True)
    api.context().set_option("fixed_seed", 0)
    rows = []
    for _, kw in SHAPES:   # every shape before the first capture: a captured workspace never grows
        api.reserve_backward_async(1, kw["E"], kw["H"], kw["W"], kw["M"], kw["sub"])
    for label, kw in SHAPES:
        sc = make_scene(seed=7, **kw)
        E, H, W, M, sub = kw["E"], kw["H"], kw["W"], kw["M"], kw["sub"]
        coords = torch.from_numpy(sc.coords).cuda()
        grads = torch.zeros_like(coords)
        assign = torch.from_numpy(sc.assign).cuda()
        shifts = torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda")
        cams = torch.tensor([sc.f, sc.ppx, sc.ppy], device="cuda")
        d_scores = torch.randn(M, dtype=torch.float64, device="cuda")
        d_poses = torch.randn(M, 6, dtype=torch.float64, device="cuda")
        tape = torch.zeros(api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, device="cuda")
        scores = torch.zeros(M, dtype=torch.float64, device="cuda")
        poses = torch.zeros(M, 6, dtype=torch.float64, device="cuda")
        contrib = torch.zeros(M, dtype=torch.bool, device="cuda")
        fstatus = torch.zeros((), dtype=torch.int32, device="cuda")
        bstatus = torch.zeros((), dtype=torch.int32, device="cuda")

        def eager():
            _, _, _, t = api.hypotheses_forward(coords, assign, *sc.params)
            api.hypotheses_backward(t, coords, grads, d_scores, d_poses)

        def stream_ordered():
            api.hypotheses_forward_async(coords, assign, shifts, cams, *TAIL, sub, tape, scores, poses, contrib, fstatus)
            api.hypotheses_backward_async(tape, coords, grads, M, d_scores, d_poses, bstatus)

        for _ in range(3):
            eager()
            stream_ordered()
        torch.cuda.synchronize()
        st = api.last_stats()
        g = capture(stream_ordered)
        step_eager, step_graph, step_inputs = training_steps(sc, E, M, sub)
        res = {"shape": label, "n_contrib": st["n_contrib"]}
        for kind, fn in (("eager", eager), ("async", stream_ordered), ("graph", g.replay), ("step_eager", step_eager),
                         ("step_graph", step_graph.replay)):
            res[kind] = timed(fn, R)
        torch.cuda.synchronize()
        assert int(fstatus) == 0 and int(bstatus) == 0
        rows.append(res)
        print(f"{label:26s} contributing {st['n_contrib']:4d} | host ms/image: eager {res['eager'][0]:7.3f} async "
              f"{res['async'][0]:7.3f} graph {res['graph'][0]:7.3f} step eager {res['step_eager'][0]:7.3f} step graph "
              f"{res['step_graph'][0]:7.3f} | device ms/image: eager {res['eager'][1]:7.3f} async {res['async'][1]:7.3f} "
              f"graph {res['graph'][1]:7.3f} step eager {res['step_eager'][1]:7.3f} step graph {res['step_graph'][1]:7.3f}",
              flush=True)
        del g, step_graph, step_inputs
    if opt.json:
        Path(opt.json).write_text(json.dumps({"card": name, "images": R, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
