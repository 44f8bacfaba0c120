"""Time the gating network (the reference's Gating, code/gating.py) on the device, as device time per call from CUDA events:

  torch        Gating.forward in float32 (cuDNN, TF32 allowed), NCHW and channels_last, with cudnn.benchmark off and on;
  GatingNet    GatingNet.forward_async into preallocated outputs.

Cases: capacity 1 with E in {7, 19}, capacity 2 with E in {10, 50}; 480x640 and 480x853; B in {1, 8}.  Then the captured
test step per image -- gating, the hypothesis draw (api.assign_hypotheses_async), ExpertStack.forward_async and
api.forward_async, one graph replayed per image -- with the torch gating (NCHW, benchmark on) and with GatingNet, at E in
{7, 19} and 480x640, as the host clock around the replays over the image count.  The card's name and power limit are
read in the same process.

    python tools/gating_timing.py --iters 50 --json /tmp/gating_timing.json
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import esac_b200.api as api  # noqa: E402
from esac_b200.compat import OUTPUT_SUBSAMPLE  # noqa: E402
from esac_b200.experts import ExpertStack, prediction_size  # noqa: E402
from esac_b200.gating_net import GatingNet, layers  # noqa: E402
from oracle import expert_oracle as XO  # noqa: E402
from oracle import gating_oracle as O  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def gflop(E: int, c: int, H: int, W: int) -> float:
    """GFLOP of one image: 2 * Hout * Wout * Cout * Cin * k * k per convolution (fc layers at 1x1)."""
    total, h, w = 0.0, H, W
    for name, cin, cout, k, s in layers(E, c):
        if name.startswith("fc"):
            h = w = 1
        elif s == 2:
            h, w = (h + 1) // 2, (w + 1) // 2
        total += 2.0 * h * w * cout * cin * k * k
    return total / 1e9


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


def torch_gating(sd, E, c, dev, channels_last=False):
    m = O.make_gating_class()(E, c).to(dev).eval()
    m.load_state_dict(sd)
    return m.to(memory_format=torch.channels_last) if channels_last else m


def kernel_rows(iters: int, dev) -> list:
    rows = []
    for c, Es in ((1, (7, 19)), (2, (10, 50))):
        for E in Es:
            sd = O.kaiming_state_dict(E, E, c)
            net = GatingNet(sd, dev)
            m, m_cl = torch_gating(sd, E, c, dev), torch_gating(sd, E, c, dev, channels_last=True)
            for H, W in ((480, 640), (480, 853)):
                for B in (1, 8):
                    g = torch.Generator().manual_seed(H + W + B)
                    img = ((torch.rand((B, 3, H, W), generator=g) - 0.4) / 0.25).to(dev)
                    img_cl = img.contiguous(memory_format=torch.channels_last)
                    out = torch.empty((B, E), device=dev)
                    probs = torch.empty((B, E), device=dev)
                    net.reserve(B, H, W)
                    row = {"c": c, "E": E, "H": H, "W": W, "B": B, "gflop_per_image": round(gflop(E, c, H, W), 3)}
                    with torch.no_grad():
                        for bench in (False, True):
                            torch.backends.cudnn.benchmark = bench
                            tag = "bench" if bench else "nobench"
                            row[f"torch_nchw_{tag}_ms"] = round(device_ms(lambda: m(img), iters), 4)
                            row[f"torch_cl_{tag}_ms"] = round(device_ms(lambda: m_cl(img_cl), iters), 4)
                        row["gatingnet_ms"] = round(device_ms(lambda: net.forward_async(img, out, probs), iters), 4)
                    best = min(v for k, v in row.items() if k.startswith("torch_"))
                    row["best_torch_over_gatingnet"] = round(best / row["gatingnet_ms"], 2)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
            del net
            torch.cuda.empty_cache()
    return rows


def step_rows(images: int, dev) -> list:
    """The captured test step per image, torch gating against GatingNet."""
    rows = []
    H, W, M = 480, 640, 256
    h, w = prediction_size(H, W)
    thresholds = (10.0, 100.0, 0.5, 100.0, OUTPUT_SUBSAMPLE)          # test_esac.py:32-41
    torch.backends.cudnn.benchmark = True
    api.reserve_forward_async(1, 19, h, w, M, OUTPUT_SUBSAMPLE)   # the largest case, before the first capture
    for E in (7, 19):
        sd = O.kaiming_state_dict(E, E, 1)
        stack = ExpertStack([XO.kaiming_state_dict(10 + e, mean=(float(e), 0.0, 2.0)) for e in range(E)], dev)
        stack.reserve(1, H, W)
        row = {"E": E, "H": H, "W": W, "images": images}
        for route in ("torch", "gatingnet"):
            m = torch_gating(sd, E, 1, dev)
            net = GatingNet(sd, dev)
            net.reserve(1, H, W)
            image = torch.zeros(1, 3, H, W, device=dev)
            camera = torch.tensor([525.0, W / 2, H / 2], device=dev)
            shift = torch.zeros(2, dtype=torch.int32, device=dev)
            seed = torch.tensor([777], dtype=torch.int64, device=dev)
            e_hyps = torch.zeros(M, dtype=torch.int64, device=dev)
            hist = torch.zeros(1, E, device=dev)
            draw_status = torch.zeros((), dtype=torch.int32, device=dev)
            log_p = torch.zeros(1, E, device=dev)
            probs = torch.zeros(1, E, device=dev)
            prediction = torch.zeros(1, E, 3, h, w, device=dev)
            pose = torch.zeros(4, 4, device=dev)
            expert = torch.zeros((), dtype=torch.int64, device=dev)
            status = torch.zeros((), dtype=torch.int32, device=dev)

            def step():
                with torch.no_grad():
                    if route == "torch":
                        probs.copy_(torch.exp(m(image)))
                    else:
                        net.forward_async(image, log_p, probs)
                    api.assign_hypotheses_async(probs[0], M, seed, e_hyps, hist[0], draw_status, maxExperts=2)
                    seed.add_(1)
                    stack.forward_async(image, hist, prediction)
                api.forward_async(prediction[0], e_hyps, shift, camera, *thresholds, pose, expert, status)

            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                step()
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step()
            gen = torch.Generator().manual_seed(5)
            frames = [((torch.rand((1, 3, H, W), generator=gen) - 0.4) / 0.25).to(dev) for _ in range(4)]
            for f in frames:                                   # warm-up
                image.copy_(f)
                graph.replay()
            torch.cuda.synchronize()
            total = 0.0
            for i in range(images):
                image.copy_(frames[i % len(frames)])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                graph.replay()
                torch.cuda.synchronize()
                total += time.perf_counter() - t0
            row[f"step_{route}_ms"] = round(1e3 * total / images, 3)
            del graph
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--images", type=int, default=40)
    ap.add_argument("--json", type=str, default="")
    opt = ap.parse_args(argv)
    torch.backends.cudnn.allow_tf32 = True
    dev = torch.device("cuda")
    info = card()
    print(json.dumps(info), flush=True)
    rows = kernel_rows(opt.iters, dev)
    steps = step_rows(opt.images, dev)
    if opt.json:
        Path(opt.json).parent.mkdir(parents=True, exist_ok=True)
        Path(opt.json).write_text(json.dumps({"card": info, "rows": rows, "steps": steps}, indent=1))


if __name__ == "__main__":
    main()
