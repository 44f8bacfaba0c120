"""Pure prefilter throughput: ONE wave with a 2048-try window for every hypothesis (3.67 M tries in one launch per lane)."""
import sys
sys.path.insert(0, str(__import__('pathlib').Path(__file__).resolve().parents[1]))
import numpy as np, torch
import esac_b200.api as api
from esac_b200.synth import make_scene
ctx = api.context()
ctx.set_option("fixed_seed", 1)
sc = make_scene(E=7, H=480, W=640, M=256, sub=1, seed=0, per_expert=True, active_only=False)
co, asg = torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda()
out = torch.zeros(4, 4, device="cuda")
for lanes in (1, 2):
    ctx.set_option("sample_groups", lanes); ctx.set_option("sample_trace", 1)
    ctx.set_option("sample_span0", 2048); ctx.set_option("sample_waves", 1); ctx.set_option("max_tries", 2048)
    for rep in range(3):
        ctx.set_seed(100 + rep)
        api.forward(co, asg, out, *sc.params)
    tr = ctx.sample_trace()
    pr = ctx.sample_profile()
    for g in range(lanes):
        p0, p1, e0, e1 = (tr[g, 0, 0, 0], tr[g, 0, 0, 1], tr[g, 0, 1, 0], tr[g, 0, 1, 1])
        print(f"lanes {lanes} lane {g}: prefilter {p0/1e3:.1f} -> {p1/1e3:.1f} us ({(p1-p0)/1e3:.1f})  exact {(e1-e0)/1e3:.1f} us; tries total {pr['tries_prefiltered']} survivors {pr['survivors_judged']}")
