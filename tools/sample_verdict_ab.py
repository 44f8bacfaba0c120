"""Where the sampling stage's time goes under the shipping options (GPU only): per lane and wave, the prefilter and exact
(verdict) kernels' first-CTA start / last-CTA end from option sample_trace, the gaps between them, and the stage's
counters (tries the sequential loop needs, tries prefiltered, survivors judged), on the bench scenes (7 experts x 256
hypotheses, 480x640).  tools/sample_profile.py compares window policies; this script traces the shipping one.

    python tools/sample_verdict_ab.py [--tree DIR] [--reps N] [--set key=value ...] [--json OUT]

--tree imports esac_b200 from another checkout (built in place), so two builds can be traced in one job.  --set overrides
a sampling option (sample_span0, sample_window, sample_waves, sample_groups, sample_tail_boost) for a sweep; the stage time
(ms_sample) is then measured with the trace off, since stamping adds atomics to every CTA."""
import argparse
import json
import sys
from pathlib import Path

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=str(Path(__file__).resolve().parents[1]))
ap.add_argument("--reps", type=int, default=8)
ap.add_argument("--set", action="append", default=[], metavar="KEY=VALUE")
ap.add_argument("--json", default=None)
args = ap.parse_args()
sys.path.insert(0, str(Path(args.tree).resolve()))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import esac_b200.api as api  # noqa: E402
from esac_b200.synth import make_scene  # noqa: E402

SHIPPING = {"sample_span0": 256, "sample_window": 1.25, "sample_waves": 6, "sample_groups": 2, "sample_tail_boost": 1.0}
opts = dict(SHIPPING)
for kv in args.set:
    k, v = kv.split("=")
    opts[k] = float(v)

ctx = api.context()
ctx.set_option("fixed_seed", 1)
for k, v in opts.items():
    ctx.set_option(k, v)
# the bench scenes: bench.py's first two images of rank 0
scs = [make_scene(E=7, H=480, W=640, M=256, sub=1, seed=s, per_expert=True, active_only=False) for s in (0, 1)]
dev = [(torch.from_numpy(sc.coords).cuda(), torch.from_numpy(sc.assign).cuda(), sc) for sc in scs]
out = torch.zeros(4, 4, device="cuda")


def run(rep):
    co, asg, sc = dev[rep % 2]
    ctx.set_seed(100 + rep)
    api.forward(co, asg, out, *sc.params)
    torch.cuda.synchronize()


# stage time and counters with the trace off
ctx.set_option("sample_trace", 0)
for rep in range(4):
    run(rep)
ms, rows = [], []
for rep in range(args.reps):
    run(rep)
    st, pr = ctx.stats(), ctx.sample_profile()
    ms.append(st["ms_sample"])
    rows.append((int(ctx.hypotheses()["tries"].sum()), pr["tries_prefiltered"], pr["survivors_judged"], pr["waves"],
                 pr["left_to_tail"]))
r = np.array(rows, float).mean(0)
summary = {"tree": str(Path(args.tree).resolve()), "options": opts, "gpu": torch.cuda.get_device_name(0),
           "ms_sample_mean": float(np.mean(ms)), "ms_sample_min": float(np.min(ms)), "ms_sample_max": float(np.max(ms)),
           "tries_needed": r[0], "tries_prefiltered": r[1], "survivors_judged": r[2], "waves": r[3], "left_to_tail": r[4]}

# timeline of one forward per scene, trace on
ctx.set_option("sample_trace", 1)
tables = []
for rep in range(2):
    run(rep)
    run(rep)  # the second call of the same scene and seed is the one stamped
    tr = ctx.sample_trace()
    lines, pre_us, ex_us = [], 0.0, 0.0
    for g in range(4):
        prev_end = None
        for w in range(32):
            if tr[g, w, 0, 0] < 0:
                continue
            p0, p1, e0, e1 = (tr[g, w, k, j] / 1e3 for k in (0, 1) for j in (0, 1))
            gap_in = p0 - prev_end if prev_end is not None else 0.0
            lines.append({"lane": g, "wave": w, "pre_start": p0, "pre_end": p1, "exact_start": e0, "exact_end": e1,
                          "pre_us": p1 - p0, "gap_pre_exact_us": e0 - p1, "exact_us": e1 - e0, "gap_from_prev_wave_us": gap_in})
            pre_us += p1 - p0
            ex_us += e1 - e0
            prev_end = e1
    tables.append({"scene": rep, "ms_sample_traced": ctx.stats()["ms_sample"], "waves": lines,
                   "sum_prefilter_us": pre_us, "sum_exact_us": ex_us})
ctx.set_option("sample_trace", 0)
summary["traces"] = tables

print(f"{summary['gpu']}  tree {summary['tree']}  options {opts}")
print(f"ms_sample {summary['ms_sample_mean']:.3f} (min {summary['ms_sample_min']:.3f}, max {summary['ms_sample_max']:.3f})  "
      f"tries needed {r[0]:.0f}  prefiltered {r[1]:.0f}  survivors {r[2]:.0f}  waves {r[3]:.1f}  left to tail {r[4]:.1f}")
for t in tables:
    print(f"--- scene {t['scene']} (traced ms_sample {t['ms_sample_traced']:.3f}); us from the first stamp")
    print("lane wave | prefilter start   end   (us) | gap | exact start   end   (us)")
    for l in t["waves"]:
        print(f"{l['lane']:4d} {l['wave']:4d} | {l['pre_start']:9.1f} {l['pre_end']:7.1f} ({l['pre_us']:5.1f}) | {l['gap_pre_exact_us']:4.1f} | "
              f"{l['exact_start']:7.1f} {l['exact_end']:7.1f} ({l['exact_us']:5.1f})")
    print(f"sum prefilter {t['sum_prefilter_us']:.1f} us, sum exact {t['sum_exact_us']:.1f} us")
if args.json:
    Path(args.json).parent.mkdir(parents=True, exist_ok=True)
    Path(args.json).write_text(json.dumps(summary, indent=1))
