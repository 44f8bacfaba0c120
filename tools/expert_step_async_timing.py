"""The expert stages' losses and training steps, eager against stream-ordered and captured (GPU only).

Part 1, the loss call alone (loss and gradient), for the reprojection loss (ref_expert.py) and the scene-coordinate loss
(init_expert.py) at 60x80 sub 8 and 480x640 sub 1, B = 1 and 8; R calls end in ONE torch.cuda.synchronize():
  eager   api.reproj_loss / api.coord_loss on CUDA tensors (each synchronises inside),
  async   api.reproj_loss_async / api.coord_loss_async in a loop, uncaptured,
  graph   replays of one captured async call.
Part 2, the whole training step with a stand-in expert FCN of realistic size (a 480x640 grey image in, a 60x80 map of scene
coordinates out, output subsampling 8): forward, loss, backward and Adam; eager on autograd.reproj_loss /
coord_loss with Adam(), against replays of the step captured on reproj_loss_async / coord_loss_async with
Adam(capturable=True).
Reported per call or step: host wall time over the R calls, and device time between CUDA events around them.  The card's
name, power limit and maximum SM clock are read in the same run.  Last, tools/reproj_bandwidth.py runs in the same process
tree (the reprojection kernel's achieved bandwidth).

    python tools/expert_step_async_timing.py [--images 200] [--json out.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import esac_b200.api as api  # noqa: E402
from backward_async_timing import capture, card, timed  # noqa: E402
from esac_b200.autograd import coord_loss, coord_loss_async, reproj_loss, reproj_loss_async  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

CUT_REPROJ, CUT_COORD = 10.0, 100.0
SHAPES = [("60x80 sub 8", 60, 80, 8), ("480x640 sub 1", 480, 640, 1)]


def expert_fcn():
    """A fully convolutional expert of the size the reference trains: three stride-2 stages to 1/8 resolution, then 3x3 and
    1x1 layers up to 512 channels and a 1x1 head to three coordinates."""
    layers, c = [], 1
    for out, k, s in ((32, 3, 1), (64, 3, 2), (128, 3, 2), (256, 3, 2), (256, 3, 1), (256, 1, 1), (512, 3, 1), (512, 1, 1),
                      (512, 1, 1), (512, 1, 1)):
        layers += [nn.Conv2d(c, out, k, s, k // 2), nn.ReLU()]
        c = out
    layers.append(nn.Conv2d(c, 3, 1))
    return nn.Sequential(*layers)


def loss_inputs(B, H, W, sub):
    sc = make_scene(E=1, H=H, W=W, M=8, sub=sub, seed=5)
    pred = torch.from_numpy(sc.coords[0]).cuda().unsqueeze(0).repeat(B, 1, 1, 1).contiguous()
    pred += 0.01 * torch.randn_like(pred)
    gt_coords = (pred + 0.5 * torch.randn_like(pred)).contiguous()
    gt_coords[:, :, ::4, ::3] = 0.0
    gts = torch.from_numpy(sc.gt_pose).cuda().unsqueeze(0).repeat(B, 1, 1).contiguous()
    shifts = torch.tensor([[1, -1]] * B, dtype=torch.int32, device="cuda")
    cams = torch.tensor([[525.0, W * sub / 2, H * sub / 2]] * B, device="cuda")
    return pred, gt_coords, gts, shifts, cams


def loss_rows(R):
    rows = []
    for label, H, W, sub in SHAPES:
        for B in (1, 8):
            pred, gt_coords, gts, shifts, cams = loss_inputs(B, H, W, sub)
            grads = torch.empty_like(pred)
            losses = torch.zeros(B, dtype=torch.float64, device="cuda")
            status = torch.zeros(B, dtype=torch.int32, device="cuda")
            counts = torch.zeros(B, dtype=torch.int64, device="cuda")
            calls = {
                "reproj": (lambda: api.reproj_loss(pred, gts, 525.0, 1, -1, CUT_REPROJ, sub, outGradients=grads),
                           lambda: api.reproj_loss_async(pred, gts, shifts, cams, CUT_REPROJ, sub, losses, status,
                                                         outGradients=grads)),
                "coord": (lambda: api.coord_loss(pred, gt_coords, CUT_COORD, outGradients=grads),
                          lambda: api.coord_loss_async(pred, gt_coords, CUT_COORD, losses, outGradients=grads,
                                                       outCounts=counts)),
            }
            for loss, (eager, stream_ordered) in calls.items():
                for _ in range(3):
                    eager()
                    stream_ordered()
                g = capture(stream_ordered)
                res = {"loss": loss, "shape": label, "B": B}
                for kind, fn in (("eager", eager), ("async", stream_ordered), ("graph", g.replay)):
                    res[kind] = timed(fn, R)
                torch.cuda.synchronize()
                assert int(status.max()) == 0
                rows.append(res)
                print(f"{loss:6s} {label:14s} B={B} | host us/call: eager {res['eager'][0] * 1e3:8.1f} async "
                      f"{res['async'][0] * 1e3:8.1f} graph {res['graph'][0] * 1e3:8.1f} | device us/call: eager "
                      f"{res['eager'][1] * 1e3:8.1f} async {res['async'][1] * 1e3:8.1f} graph {res['graph'][1] * 1e3:8.1f}",
                      flush=True)
                del g
    return rows


def step_rows(R):
    H, W, sub = 60, 80, 8
    image = torch.rand(1, 1, H * sub, W * sub, device="cuda")
    _, gt_coords, gts, shifts, cams = loss_inputs(1, H, W, sub)
    steps = {
        "ref_expert (reproj)": (lambda p: reproj_loss(p, gts, 525.0, 1, -1, CUT_REPROJ, sub),
                                lambda p: reproj_loss_async(p, gts, shifts, cams, CUT_REPROJ, sub)),
        "init_expert (coord)": (lambda p: coord_loss(p, gt_coords, CUT_COORD),
                                lambda p: coord_loss_async(p, gt_coords, CUT_COORD)),
    }
    rows = []
    for name, (eager_loss, async_loss) in steps.items():
        torch.manual_seed(0)
        e_net = expert_fcn().cuda()
        e_opt = torch.optim.Adam(e_net.parameters(), lr=1e-6)
        torch.manual_seed(0)
        g_net = expert_fcn().cuda()
        g_opt = torch.optim.Adam(g_net.parameters(), lr=torch.tensor(1e-6, device="cuda"), capturable=True)

        def eager():
            e_opt.zero_grad(set_to_none=False)
            eager_loss(e_net(image)).backward()
            e_opt.step()

        def captured():
            async_loss(g_net(image)).backward()
            g_opt.step()

        for _ in range(3):
            eager()
        g = capture(captured, lambda: g_opt.zero_grad(set_to_none=False))
        res = {"step": name, "parameters": sum(p.numel() for p in e_net.parameters())}
        for kind, fn in (("eager", eager), ("graph", g.replay)):
            res[kind] = timed(fn, R)
        rows.append(res)
        print(f"step {name:20s} ({res['parameters'] / 1e6:.1f} M parameters) | host ms/step: eager {res['eager'][0]:7.3f} "
              f"graph {res['graph'][0]:7.3f} | device ms/step: eager {res['eager'][1]:7.3f} graph {res['graph'][1]:7.3f}",
              flush=True)
        del g
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", "-R", type=int, default=200)
    ap.add_argument("--json", help="also write the tables here")
    opt = ap.parse_args()
    name = card()
    print(f"card (name, power limit, max SM clock): {name}", flush=True)
    api.reserve_loss_async(8, 480, 640)   # every shape before the first capture: a captured workspace never grows
    losses = loss_rows(opt.images)
    steps = step_rows(max(opt.images // 4, 20))
    if opt.json:
        Path(opt.json).write_text(json.dumps({"card": name, "calls": opt.images, "losses": losses, "steps": steps}, indent=1))
    print("tools/reproj_bandwidth.py:", flush=True)
    r = subprocess.run([sys.executable, str(Path(__file__).resolve().parent / "reproj_bandwidth.py")], capture_output=True,
                       text=True)
    print(r.stdout + r.stderr, flush=True)
    return r.returncode


if __name__ == "__main__":
    sys.exit(main())
