"""Class-wise comparison of a scene-coordinate gradient with the oracle's (oracle/esac_oracle.py backward / hypotheses_vjp).

The gradient has three kinds of cells whose sizes differ by orders of magnitude:
  minimal  cells of a contributing hypothesis's minimal set: the dPNP support term (central differences through P3P), nearly
           always the largest entries;
  inlier   final inlier cells of a contributing hypothesis: path I, -pinv(J^T J) J^T dProjectdObj through the refinement, plus
           the score term;
  rest     every other cell: the direct dScore term only.
A bar relative to the largest entry (1e-3 of max|g_ref|) is set by a minimal-set cell and hardly constrains the other two, so
each class is held to its own largest reference entry.  Cells are classed per (expert, y, x) in that order of precedence.
"""
import numpy as np

from oracle import esac_oracle as O

MINIMAL, INLIER, REST = 0, 1, 2
NAMES = ("minimal", "inlier", "rest")
FLOOR = 1e-7        # class scales are floored at this fraction of the global maximum (a class may be all but zero)
GLOBAL_BAR = 1e-3   # the bar relative to the largest entry, kept: it still guards the minimal-set cells
CAP = 1e-4          # no class-wise bar is looser than this
# the forced scene's bars (tests/test_gpu_backward.py, every refinement walk and scoring shape): about 10x the worst class
# measured on an H100 SXM (80 GB, 700 W) -- minimal 1.32e-6, inlier 1.67e-6, rest 1.80e-6.  tests/test_grad_terms.py shows
# that an error in any one term (path I, dScore, dPNP support) fails them
FORCED_BARS = {"minimal": 1.5e-5, "inlier": 2e-5, "rest": 2e-5}


def cell_classes(shape, assign, trace):
    """int8 [E,H,W] class of every cell from an oracle trace (BackwardTrace): minimal > inlier > rest."""
    E, _, H, W = shape
    cls = np.full((E, H, W), REST, np.int8)
    contrib = np.nonzero(np.asarray(trace.probs) >= O.PROB_THRESH)[0]
    for h in contrib:
        im = trace.inlier_maps[h]
        if im is not None:
            cls[int(assign[h])][im > 0] = INLIER
    for h in contrib:
        for x, y in trace.hyps[h].cells:
            cls[int(assign[h]), y, x] = MINIMAL
    return cls


def compare(g, g_ref, classes):
    """Per class: cells, max|g - g_ref| (over the three channels of its cells), the class scale max(max|g_ref|, FLOOR x global
    maximum) and their ratio; 'global' is the old bar's ratio max|g - g_ref| / max|g_ref|."""
    g = np.asarray(g, np.float64)
    g_ref = np.asarray(g_ref, np.float64)
    diff = np.abs(g - g_ref).max(axis=1)
    mag = np.abs(g_ref).max(axis=1)
    gmax = max(float(mag.max()), 1e-30)
    rep = {"global": {"cells": int(classes.size), "err": float(diff.max()), "scale": gmax, "rel": float(diff.max()) / gmax}}
    for c, name in enumerate(NAMES):
        m = classes == c
        n = int(m.sum())
        if n == 0:
            rep[name] = {"cells": 0, "err": 0.0, "scale": 0.0, "rel": 0.0}
            continue
        scale = max(float(mag[m].max()), FLOOR * gmax)
        err = float(diff[m].max())
        rep[name] = {"cells": n, "err": err, "scale": scale, "rel": err / scale}
    return rep


def fmt(rep):
    return "; ".join(f"{k}: {v['rel']:.2e} ({v['err']:.2e} of {v['scale']:.2e}, {v['cells']} cells)" for k, v in rep.items())


def failures(rep, bars):
    """Names of the classes whose ratio exceeds its bar (``bars``: one number or a dict by class name), and 'global' when the
    old bar (GLOBAL_BAR of the largest entry) fails."""
    if not isinstance(bars, dict):
        bars = {n: bars for n in NAMES}
    bad = [n for n in NAMES if rep[n]["rel"] > bars[n]]
    if rep["global"]["rel"] >= GLOBAL_BAR:
        bad.append("global")
    return bad


def assert_classwise(g, g_ref, classes, bars, what=""):
    """Asserts every class within its bar and the old global bar; returns the report."""
    rep = compare(g, g_ref, classes)
    bad = failures(rep, bars)
    assert not bad, f"{what}: {bad} over the bar {bars}: {fmt(rep)}"
    return rep


def sampled_classes(flat_idx, shape, assign, cells, probs, thresh=O.PROB_THRESH):
    """For a gradient stored as samples at flat indices of [E,3,H,W]: True where the entry's cell is in the accepted minimal set
    (cells [M,4,2] as (x, y)) of a hypothesis with probs >= thresh."""
    E, _, H, W = shape
    in_set = np.zeros((E, H, W), bool)
    for h in np.nonzero(np.asarray(probs) >= thresh)[0]:
        for x, y in cells[h]:
            in_set[int(assign[h]), int(y), int(x)] = True
    e, _, y, x = np.unravel_index(np.asarray(flat_idx), shape)
    return in_set[e, y, x]
