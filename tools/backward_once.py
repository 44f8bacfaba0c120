"""Two esac.backward calls at the bench shape (GPU only) -- the target of a profiler's launch list (per-kernel durations
of the backward's stages)."""
import sys
sys.path.insert(0, str(__import__('pathlib').Path(__file__).resolve().parents[1]))
import torch
import esac_b200.api as api
from esac_b200.synth import make_scene

ctx = api.context()
ctx.set_option("fixed_seed", 1)
sc = make_scene(E=7, H=480, W=640, M=256, sub=1, seed=0, per_expert=True, active_only=False)
coords = torch.from_numpy(sc.coords).cuda(); assign = torch.from_numpy(sc.assign).cuda()
gt = torch.from_numpy(sc.gt_pose)
grads = torch.zeros_like(coords)
for i in range(int(sys.argv[1]) if len(sys.argv) > 1 else 2):
    ctx.set_seed(7)
    loss = api.backward(coords, grads, assign, gt, 1.0, 100.0, 100.0, *sc.params)
    st = ctx.stats()
    print(f"loss {loss:.6f} contrib {st['n_contrib']} stages ms: sample {st['ms_sample']:.3f} score {st['ms_score']:.3f} refine {st['ms_refine']:.3f} "
          f"backward {st['ms_backward']:.3f} total {st['ms_total']:.3f}")
