"""Phase breakdown of one LM evaluation inside the refinement kernel (GPU only): clock64() counters of block 0."""
import sys
sys.path.insert(0, str(__import__('pathlib').Path(__file__).resolve().parents[1]))
import numpy as np, torch
import esac_b200.api as api
from esac_b200.synth import make_scene

NAMES = ["produce + receive the command (Rodrigues)", "pass over the cells", "block reduce + publish",
         "wait for the group's results", "slot summation", "map sums to (rvec,tvec)", "accept/reject + LM step",
         "root: dR/dr + change of variables"]
ctx = api.context()
ctx.set_option("fixed_seed", 1)
ctx.set_option("refine_profile", 1)
mhz = 1965.0
for name, kw in (("forward 7x256 480x640", dict(E=7, H=480, W=640, M=256, sub=1, seed=0, per_expert=True, active_only=False)),
                 ("forward native 60x80 M=256", dict(E=7, H=60, W=80, M=256, sub=8, seed=0))):
    sc = make_scene(**kw)
    coords = torch.from_numpy(sc.coords).cuda(); assign = torch.from_numpy(sc.assign).cuda()
    out = torch.zeros(4, 4, device="cuda")
    for grp in (0, 74, 37):
        ctx.set_option("refine_group", grp)
        for i in range(3):
            ctx.set_seed(100 + i)
            api.forward(coords, assign, out, *sc.params)
        st = ctx.stats()
        p = ctx.refine_profile()
        n = max(int(p[8]), 1)
        tot = p[:8].sum()
        print(f"{name}: group {st['refine_group']} refine {st['ms_refine']:.3f} ms, rounds {st['refine_rounds']}, {n} evaluations, "
              f"{tot / n:.0f} cycles = {tot / n / mhz:.2f} us per evaluation (block 0)")
        for i in range(8):
            print(f"    {NAMES[i]:42s} {p[i] / n:8.0f} cyc  {100.0 * p[i] / tot:5.1f} %")
    ctx.set_option("refine_group", 0)
