"""Replay time of a captured ESAC step that runs every expert against the same step with an ExpertGate, which runs only the
experts that drew hypotheses (GPU only).

The experts are tools/expert_step_async_timing.py's stand-in FCN (a 480x640 grey image in, a 60x80 map of scene
coordinates out).  Each expert's output perturbs a synthetic scene's coordinates by 1e-3 of it, so ESAC has a real map to
work on.  The draw is api.assign_hypotheses_async with M = 256 and maxExperts = k from fixed gating logits, so exactly k
of the E experts draw hypotheses; k = E (every expert active) measures what the gate itself costs.
  test step   experts forward (no grad), esac.forward (api.forward_async);
  train step  experts forward, esac_loss_async, loss.backward(), each expert's backward and Adam(capturable=True) step, the
              gating logits' Adam step (examples/train_step_gated_graph_synthetic.py's structure).
Reported: device ms per replay between CUDA events around R replays.  The card's name, power limit and maximum SM clock
are read in the same run.

    python tools/gated_step_timing.py [--replays 20] [--json out.json]
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import torch  # noqa: E402

import esac_b200.api as api  # noqa: E402
from backward_async_timing import card, timed  # noqa: E402
from esac_b200.autograd import esac_loss_async  # noqa: E402
from esac_b200.gate import ExpertGate  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402
from expert_step_async_timing import expert_fcn  # noqa: E402

H, W, SUB, M = 60, 80, 8, 256
THRESH = (10.0, 100.0, 0.5, 100.0, SUB)


class AlwaysGate:
    """Runs every region: the ungated step."""

    def arm(self, counts):
        pass

    def run(self, i, fn):
        return fn()


def init_adam_state(opt):
    """Adam's lazily created state, created before the capture (a region may be skipped by every warm-up step)."""
    for group in opt.param_groups:
        for p in group["params"]:
            if not opt.state[p]:
                opt.state[p].update(step=torch.zeros((), device=p.device), exp_avg=torch.zeros_like(p),
                                    exp_avg_sq=torch.zeros_like(p))


def make_step(E, k, gated, train):
    """The step's function, its gate and what it keeps alive."""
    torch.manual_seed(0)
    sc = make_scene(E=E, H=H, W=W, M=M, sub=SUB, seed=3, active_only=False)
    prior = torch.from_numpy(sc.coords).cuda()
    image = torch.rand(1, 1, H * SUB, W * SUB, device="cuda")
    experts = [expert_fcn().cuda() for _ in range(E)]
    logits = torch.zeros(1, E, device="cuda")
    logits[0, E - k:] = 1.0                      # the k last experts are the k most likely ones
    logits.requires_grad_(train)
    seed = torch.tensor([1], dtype=torch.int64, device="cuda")
    e_hyps = torch.zeros(M, dtype=torch.int64, device="cuda")
    hist = torch.zeros(E, device="cuda")
    st = torch.zeros((), dtype=torch.int32, device="cuda")
    shift = torch.tensor([sc.shiftX, sc.shiftY], dtype=torch.int32, device="cuda")
    camera = torch.tensor([sc.params[2], sc.params[3], sc.params[4]], device="cuda")
    gt = torch.from_numpy(sc.gt_pose).cuda()
    prediction = torch.zeros(E, 3, H, W, device="cuda")
    pose, expert, status = torch.zeros(4, 4, device="cuda"), torch.zeros((), dtype=torch.int64, device="cuda"), st.clone()
    gate = ExpertGate(E) if gated else AlwaysGate()
    opts = [torch.optim.Adam(m.parameters(), lr=1e-6, capturable=True) for m in experts] if train else []
    g_opt = torch.optim.Adam([logits], lr=1e-4, capturable=True) if train else None
    for o in opts + ([g_opt] if train else []):
        init_adam_state(o)

    def step():
        log_probs = torch.log_softmax(logits, dim=1)
        api.assign_hypotheses_async(torch.exp(log_probs).detach()[0], M, seed, e_hyps, hist, st, maxExperts=k)
        seed.add_(1)
        gate.arm(hist)
        outs = [None] * E
        with torch.no_grad():
            prediction.zero_()

        def forward(e):
            with torch.set_grad_enabled(train):
                outs[e] = experts[e](image)[0]
            with torch.no_grad():
                prediction[e].copy_(prior[e] + 1e-3 * outs[e])
        for e in range(E):
            gate.run(e, lambda e=e: forward(e))
        if not train:
            api.forward_async(prediction, e_hyps, shift, camera, *THRESH, pose, expert, status)
            return
        leaf = prediction.detach().requires_grad_()
        g_opt.zero_grad(set_to_none=True)
        loss = esac_loss_async(leaf, log_probs, e_hyps, gt, shift, camera, 1.0, 100.0, 100.0, *THRESH, status=status)
        loss.backward()

        def backward(e):
            opts[e].zero_grad(set_to_none=True)
            torch.autograd.backward(outs[e], 1e-3 * leaf.grad[e])
            opts[e].step()
        for e in range(E):
            gate.run(e, lambda e=e: backward(e))
        g_opt.step()

    return step, gate, (experts, opts, prediction, status)


def replay_ms(E, k, gated, train, R):
    step, gate, keep = make_step(E, k, gated, train)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph(keep_graph=gated)
    with torch.cuda.graph(graph):
        step()
    if gated:
        gate.finalize(graph)
    graph.replay()
    torch.cuda.synchronize()
    ms = timed(graph.replay, R)[1]
    assert int(keep[3]) == 0, "bad assignment"
    del graph
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", "-R", type=int, default=20)
    ap.add_argument("--json", help="also write the table here")
    opt = ap.parse_args()
    torch.backends.cudnn.benchmark = False
    name = card()
    print(f"card (name, power limit, max SM clock): {name}", flush=True)
    print(f"device ms per replay, R = {opt.replays}, 480x640 images, {H}x{W} maps, M = {M}", flush=True)
    api.reserve_backward_async(1, 19, H, W, M, SUB)   # the largest shape, before the first capture (covers the forward)
    rows = []
    for train in (False, True):
        for E in (4, 19):
            for k in (1, 2, E):
                ungated = replay_ms(E, k, False, train, opt.replays)
                gated = replay_ms(E, k, True, train, opt.replays)
                rows.append(dict(step="train" if train else "test", E=E, active=k, ungated_ms=ungated, gated_ms=gated))
                print(f"{'train' if train else 'test ':5s} step  E = {E:2d}, {k:2d} active: ungated {ungated:8.3f} ms, "
                      f"gated {gated:8.3f} ms ({ungated / gated:5.2f}x)", flush=True)
                torch.cuda.empty_cache()
    if opt.json:
        Path(opt.json).write_text(json.dumps({"card": name, "replays": opt.replays, "rows": rows}, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
