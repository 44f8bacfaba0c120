"""Time three routes to the predictions of k active experts out of E (the reference's Expert, code/expert.py) on one
image, each as device time per call from CUDA events:

  torch loop   the per-expert torch forward (cuDNN, default TF32), NCHW and channels_last, the better of the two;
  grouped      one torch stack of the k active experts: conv1 with their filters side by side, every later layer a
               grouped convolution (groups = k);
  stack        ExpertStack.forward with a histogram that activates the k experts.

Cases: E in {7, 19}, k in {1, 2, 4, E}, 480x640 and 480x853 images.  Achieved TFLOP/s use the FLOP count of the layer
table (2 * Hout * Wout * Cout * Cin * kh * kw per layer and active expert).  The card's name and power limit are read in
the same process.

    python tools/expert_stack_timing.py --iters 20 --json /tmp/expert_stack_timing.json
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from esac_b200.experts import LAYERS, ExpertStack  # noqa: E402
from oracle import expert_oracle as O  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def flops(H: int, W: int) -> float:
    """FLOPs of one expert on one HxW image."""
    total, h, w = 0.0, H, W
    for _, cin, cout, k, s in LAYERS:
        if s == 2:
            h, w = (h + 1) // 2, (w + 1) // 2
        total += 2.0 * h * w * cout * cin * k * k
    return total


def device_ms(fn, iters: int) -> float:
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def grouped_params(ps):
    """The k experts' parameters as one grouped network: weights and biases concatenated along Cout."""
    return {k: torch.cat([p[k] for p in ps]) for k in ps[0]}


def grouped_forward(x, g, k):
    layer = {name: (ks, s) for name, _, _, ks, s in LAYERS}

    def conv(name, v, groups=k):
        ks, s = layer[name]
        return F.conv2d(v, g[name + ".weight"], g[name + ".bias"], stride=s, padding=ks // 2, groups=groups)

    x = F.relu(conv("conv1", x, 1))
    x = F.relu(conv("conv2", x))
    x = F.relu(conv("conv3", x))
    res = F.relu(conv("conv4", x))
    x = F.relu(conv("res1_conv3", F.relu(conv("res1_conv2", F.relu(conv("res1_conv1", res))))))
    res = res + x
    x = F.relu(conv("res2_conv3", F.relu(conv("res2_conv2", F.relu(conv("res2_conv1", res))))))
    res = conv("res2_skip", res) + x
    x = F.relu(conv("res3_conv3", F.relu(conv("res3_conv2", F.relu(conv("res3_conv1", res))))))
    res = res + x
    x = conv("fc3", F.relu(conv("fc2", F.relu(conv("fc1", res)))))
    return x + g["mean"].view(1, 3 * k, 1, 1)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", type=str, default="")
    opt = ap.parse_args(argv)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda")
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    for E in (7, 19):
        sds = [O.kaiming_state_dict(e) for e in range(E)]
        stack = ExpertStack(sds, dev)
        params = [{k: v.to(dev) for k, v in sd.items()} for sd in sds]
        params_cl = [{k: (v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v) for k, v in p.items()}
                     for p in params]
        for H, W in ((480, 640), (480, 853)):
            g = torch.Generator().manual_seed(H + W)
            img = ((torch.rand((1, 3, H, W), generator=g) - 0.4) / 0.25).to(dev)
            img_cl = img.contiguous(memory_format=torch.channels_last)
            for k in sorted({1, 2, 4, E}):
                active = list(range(0, E, max(1, E // k)))[:k]
                hist = torch.zeros(1, E, device=dev)
                hist[0, active] = 1.0
                grouped = grouped_params([params[e] for e in active])
                out = torch.empty((1, E, 3, (H + 7) // 8, (W + 7) // 8), device=dev)
                stack.reserve(1, H, W)
                with torch.no_grad():
                    t_nchw = device_ms(lambda: [O.apply(img, params[e]) for e in active], opt.iters)
                    t_cl = device_ms(lambda: [O.apply(img_cl, params_cl[e]) for e in active], opt.iters)
                    t_grp = device_ms(lambda: grouped_forward(img, grouped, k), opt.iters)
                    t_stack = device_ms(lambda: stack.forward_async(img, hist, out), opt.iters)
                gf = flops(H, W) * k / 1e9
                best = min(t_nchw, t_cl, t_grp)
                row = {"E": E, "k": k, "H": H, "W": W, "gflop": round(gf, 1),
                       "torch_loop_nchw_ms": round(t_nchw, 3), "torch_loop_cl_ms": round(t_cl, 3),
                       "grouped_ms": round(t_grp, 3), "stack_ms": round(t_stack, 3),
                       "stack_tflops": round(gf / t_stack, 1), "best_torch_tflops": round(gf / best, 1),
                       "stack_speedup_vs_best_torch": round(best / t_stack, 2)}
                rows.append(row)
                print(json.dumps(row), flush=True)
        del stack
        torch.cuda.empty_cache()
    if opt.json:
        Path(opt.json).parent.mkdir(parents=True, exist_ok=True)
        Path(opt.json).write_text(json.dumps({"card": info, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
