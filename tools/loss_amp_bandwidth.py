"""The 16-bit expert losses against the float32 ones and against the prediction.float() route, on the GPU.

1. Kernel time of the eager loss calls (the library's stage timer `ms_score`: CUDA events around the loss kernels alone)
   for float32 / float16 / bfloat16 predictions, loss only and with the gradient (16-bit: scaled on the device), with the
   algorithmic bytes per cell and the achieved GB/s:
     reprojection   loss + gradient: 24 B (float32) / 12 B (16-bit)    loss only: 12 B / 6 B
     coordinates    loss + gradient: 48 B / 36 B (count pass 12 B, loss pass 24 / 18 B read + 12 / 6 B written)
                    loss only: 24 B / 18 B
2. Forward + backward of the 16-bit stream-ordered nodes against the prediction.float() route into the float32 node, each
   captured in a CUDA graph and timed over replays with CUDA events.  Algorithmic bytes per cell of the reprojection loss:
   16-bit node 18 B (forward 6 B, backward 6 + 6 B); the float32 node on the upcast output 48 B plus the cast (6 + 12 B)
   and the gradient's scale and cast back (12 + 12 + 6 B): about 84 B (3 channels throughout).
3. A replayed training step of a stand-in FCN (three convs to 3 x 60 x 80, then the reprojection loss) under
   torch.autocast in bfloat16 against the same step in float32.

Needs a GPU; prints the card name and power limit first.  Sizes: 480x640 maps at B = 8, 64, 256 and 60x80 maps."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import esac_b200.api as api  # noqa: E402
from esac_b200 import autograd as ag  # noqa: E402

PEAK_GBS = 3350.0   # H100 SXM data sheet, HBM3
CUT, SUB = 10.0, 8
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
SIZES = [(8, 480, 640), (64, 480, 640), (256, 480, 640), (64, 60, 80), (8, 60, 80)]


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def scene(B, H, W, g):
    """Scene coordinates 1-6 m in front of an identity camera near its pixels, identity poses, coordinate ground truths."""
    z = torch.rand((B, 1, H, W), device="cuda", generator=g) * 5 + 1
    ys = torch.arange(H, device="cuda").view(1, 1, H, 1) * SUB + SUB / 2 - H * SUB / 2
    xs = torch.arange(W, device="cuda").view(1, 1, 1, W) * SUB + SUB / 2 - W * SUB / 2
    noise = torch.randn((B, 2, H, W), device="cuda", generator=g) * 20
    pred = torch.cat([(xs + noise[:, :1]) * z / 500, (ys + noise[:, 1:]) * z / 500, z], 1)
    gt = pred + torch.randn((B, 3, H, W), device="cuda", generator=g) * 0.3
    gt *= torch.rand((B, 1, H, W), device="cuda", generator=g) < 0.9
    return pred, torch.eye(4, device="cuda").repeat(B, 1, 1), gt


def kernels(ctx, call, n=20):
    for _ in range(3):
        call()
    ms = []
    for _ in range(n):
        call()
        ms.append(ctx.stats()["ms_score"])
    return median(ms)


def kernel_table(ctx, g):
    print("\n1. loss kernels (ms_score), us and GB/s (share of the 3.35 TB/s data-sheet peak)")
    for B, H, W in SIZES:
        pred32, poses, gt = scene(B, H, W, g)
        cells = B * H * W
        scale = torch.full((1,), 65536.0 / B, device="cuda")
        for dt in DTYPES:
            pred = pred32.to(dt)
            grads = torch.empty_like(pred)
            amp = dt != torch.float32
            rp = api.reproj_loss_amp if amp else api.reproj_loss
            cl = api.coord_loss_amp if amp else api.coord_loss
            kw = {"gradScale": scale} if amp else {}
            rows = [("reproj loss+grad", 12 if amp else 24,
                     lambda: rp(pred, poses, 500.0, 0, 0, CUT, SUB, outGradients=grads, **kw)),
                    ("reproj loss", 6 if amp else 12, lambda: rp(pred, poses, 500.0, 0, 0, CUT, SUB)),
                    ("coord loss+grad", 36 if amp else 48, lambda: cl(pred, gt, CUT, outGradients=grads, **kw)),
                    ("coord loss", 18 if amp else 24, lambda: cl(pred, gt, CUT))]
            line = f"B={B:3d} {H}x{W} {str(dt)[6:]:8s}"
            for name, nbytes, call in rows:
                k = kernels(ctx, call)
                gbs = cells * nbytes / k / 1e6
                line += f" | {name} {nbytes:2d} B: {k * 1e3:8.1f} us {gbs:6.0f} GB/s ({gbs / PEAK_GBS:.2f})"
            print(line, flush=True)
        del pred32, gt


def replay_ms(fn, n=30):
    """fn (forward + backward) captured in a CUDA graph, ms per replay over n replays (CUDA events)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(3):
        g.replay()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        g.replay()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / n


def node_table(g):
    print("\n2. forward + backward of the stream-ordered reprojection node, one CUDA graph replay, us")
    api.reserve_loss_async(max(B for B, _, _ in SIZES), 480, 640)   # before the first capture
    for B, H, W in SIZES:
        pred32, poses, _ = scene(B, H, W, g)
        shifts = torch.zeros(B, 2, dtype=torch.int32, device="cuda")
        cams = torch.tensor([[500.0, W * SUB / 2, H * SUB / 2]] * B, device="cuda")
        line = f"B={B:3d} {H}x{W}"
        for dt in (torch.float16, torch.bfloat16):
            p = pred32.to(dt).requires_grad_()

            def amp():
                p.grad = None
                ag.reproj_loss_async(p, poses, shifts, cams, CUT, SUB).backward()

            def upcast():
                p.grad = None
                ag.reproj_loss_async(p.float(), poses, shifts, cams, CUT, SUB).backward()

            a, u = replay_ms(amp), replay_ms(upcast)
            line += f" | {str(dt)[6:]}: 16-bit node {a * 1e3:8.1f} us, p.float() route {u * 1e3:8.1f} us ({u / a:.2f}x)"
            del p
        print(line, flush=True)
        del pred32


def step_table():
    print("\n3. stand-in FCN training step (forward, reprojection loss, backward), one CUDA graph replay, ms")
    for B in (8, 64):
        torch.manual_seed(0)
        net = torch.nn.Sequential(torch.nn.Conv2d(3, 32, 3, stride=2, padding=1), torch.nn.ReLU(),
                                  torch.nn.Conv2d(32, 64, 3, stride=2, padding=1), torch.nn.ReLU(),
                                  torch.nn.Conv2d(64, 3, 3, stride=2, padding=1)).cuda()
        image = torch.randn(B, 3, 480, 640, device="cuda")
        g = torch.Generator(device="cuda").manual_seed(1)
        target, poses, _ = scene(B, 60, 80, g)
        shifts = torch.zeros(B, 2, dtype=torch.int32, device="cuda")
        cams = torch.tensor([[500.0, 320.0, 240.0]] * B, device="cuda")
        res = {}
        for name, dt in (("float32", None), ("bfloat16 autocast", torch.bfloat16)):
            def step():
                net.zero_grad(set_to_none=False)
                with torch.autocast("cuda", dtype=dt or torch.float32, enabled=dt is not None):
                    p = net(image)
                    p.add_(target)
                    loss = ag.reproj_loss_async(p, poses, shifts, cams, CUT, SUB)
                loss.backward()
            res[name] = replay_ms(step)
        print(f"B={B:3d} 480x640 image -> 60x80 map: float32 {res['float32']:.3f} ms, bfloat16 autocast "
              f"{res['bfloat16 autocast']:.3f} ms ({res['float32'] / res['bfloat16 autocast']:.2f}x)", flush=True)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("loss_amp_bandwidth: no CUDA device")
    print(f"card: {card()}")
    ctx = api.context()
    g = torch.Generator(device="cuda").manual_seed(5)
    kernel_table(ctx, g)
    node_table(g)
    step_table()
    print(f"\ncard: {card()}")


if __name__ == "__main__":
    main()
