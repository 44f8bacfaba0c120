"""The oracle's hypotheses node (oracle/esac_oracle.py hypotheses_vjp) at any probability floor.

The oracle gates every hypothesis on p >= PROB_THRESH.  With an upstream gradient given, d_sm_score and assemble read the
probabilities only for that gate, so passing them a 0 / 1 gate in place of p differentiates exactly the hypotheses with
!(p < prob_thresh); the refinement loop is _refined_hypotheses's with the same test.  With prob_thresh = PROB_THRESH
the result is hypotheses_vjp's bit for bit (tests/test_floor_oracle.py)."""
from types import SimpleNamespace

import numpy as np

from oracle import esac_oracle as O


def gate(probs, prob_thresh):
    """1.0 for the hypotheses with !(p < prob_thresh), else 0.0: what the oracle's `p < PROB_THRESH` tests see."""
    return np.where(np.asarray(probs, np.float64) < prob_thresh, 0.0, 1.0)


def refined_hypotheses(coords, assign, sampling, K, tau, alpha, beta, max_reproj, seed, prob_thresh,
                       max_tries=O.MAX_SAMPLING_TRIES, injected_cells=None, mt=None):
    """_refined_hypotheses with the refinement of every hypothesis with !(p < prob_thresh)."""
    hyps = O.sample_hypotheses(coords, assign, sampling, K, max_tries, tau, seed, injected_cells, mt)
    errs, jacs = [], []
    for h, hy in enumerate(hyps):
        e_, j_ = O.get_repro_errs(coords, hy.rvec, hy.tvec, int(assign[h]), sampling, K, max_reproj, True)
        errs.append(e_); jacs.append(j_)
    scores = O.get_hyp_scores(errs, tau, alpha, beta)
    probs = O.softmax(scores)
    ref, imaps = [], []
    for h, hy in enumerate(hyps):
        if probs[h] < prob_thresh:
            ref.append((hy.rvec.copy(), hy.tvec.copy())); imaps.append(None)
            continue
        r, t, im, _ = O.refine_hyp(coords, errs[h], sampling, K, int(assign[h]), tau, O.MAX_REF_STEPS, max_reproj,
                                   hy.rvec, hy.tvec)
        ref.append((r, t)); imaps.append(im)
    return hyps, errs, jacs, scores, probs, ref, imaps


def hypotheses_vjp(coords, assign, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, max_reproj, sub, seed, grad_poses,
                   grad_scores, prob_thresh=O.PROB_THRESH, injected_cells=None, max_tries=O.MAX_SAMPLING_TRIES, mt=None,
                   clamp_thresh=10.0):
    """O.hypotheses_vjp with the floor prob_thresh.  Returns (gradient f32 [E,3,H,W], BackwardTrace); the trace's probs are
    the softmax probabilities, its mult is 1 and its `gate` attribute the 0 / 1 contributing flags."""
    coords = np.asarray(coords)
    assign = np.asarray(assign)
    H, W = coords.shape[2], coords.shape[3]
    N = H * W
    M = len(assign)
    grad_poses = np.zeros((M, 6)) if grad_poses is None else np.asarray(grad_poses, np.float64).reshape(M, 6)
    grad_scores = np.zeros(M) if grad_scores is None else np.asarray(grad_scores, np.float64).reshape(M)
    K = O.cam_mat(f, ppx, ppy)
    sampling = O.create_sampling(W, H, sub, shiftX, shiftY)
    hyps, errs, jacs, scores, probs, ref, imaps = refined_hypotheses(coords, assign, sampling, K, tau, alpha, beta,
                                                                     max_reproj, seed, prob_thresh, max_tries,
                                                                     injected_cells, mt)
    on = gate(probs, prob_thresh)
    grad_I = [None] * M
    clamped_jr, clamped_dpnp = [], []
    for h in range(M):
        if not on[h]:
            continue
        dHyp, clamped = O.d_hyp_d_obj(coords, int(assign[h]), sampling, K, ref[h][0], ref[h][1], imaps[h], max_reproj,
                                      clamp_thresh)
        if clamped:
            clamped_jr.append(h)
        if dHyp is None:
            dHyp = np.zeros((6, N * 3))
        grad_I[h] = (grad_poses[h].reshape(1, 6) @ dHyp).reshape(N, 3)
    support = []
    grad_II = O.d_sm_score(coords, assign, sampling, hyps, None, on, errs, jacs, K, alpha, beta, tau, max_reproj,
                           clamp_thresh, clamped_dpnp, g=grad_scores, support_log=support)
    out = np.zeros(coords.shape, np.float32)
    mult = np.ones(M)
    O.assemble(out, assign, on, mult, grad_I, grad_II)
    tr = O.BackwardTrace(hyps, scores, probs, ref, imaps, None, grad_I, grad_II, clamped_jr, clamped_dpnp, support, mult)
    tr.gate = on
    return out, tr


def cell_classes(shape, assign, trace):
    """grad_terms.cell_classes for a floor trace: the contributing hypotheses are those of trace.gate."""
    import grad_terms as GT
    return GT.cell_classes(shape, assign, SimpleNamespace(probs=trace.gate, inlier_maps=trace.inlier_maps, hyps=trace.hyps))
