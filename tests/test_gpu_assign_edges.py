"""The device-side hypothesis assignment (api.assign_hypotheses / assign_hypotheses_async, gating.cu) at its edges (run with
`-m gpu`): bitwise the oracle on every input of tests/test_assign_semantics.py, the same refusals as torch.multinomial
(a NaN kept by the maxExperts clamp included), ties as the stable sort leaves them, the 1024-expert bound, its histogram
against torch.histc of its own draws, and -- independent of the oracle's algorithm -- a G-test of the drawn counts
against the float64 probabilities of the clamped weights."""
import numpy as np
import pytest
import torch

import esac_b200.api as api
from oracle import esac_oracle as O
from test_assign_semantics import BAD_ENTRY, IDS, MESSAGES, OK, PARAMS, ZERO_SUM, oracle_verdict, torch_clamp, weights

pytestmark = pytest.mark.gpu

M, SEED = 256, 2024


def _async(probs, m, seed, **kw):
    lead = tuple(probs.shape[:-1])
    a = torch.full(lead + (m,), -1, dtype=torch.int64, device="cuda")
    h = torch.full(lead + (probs.shape[-1],), -1.0, device="cuda")
    s = torch.full(lead, -7, dtype=torch.int32, device="cuda")
    api.assign_hypotheses_async(probs, m, torch.tensor([seed], dtype=torch.int64, device="cuda"), a, h, s, **kw)
    torch.cuda.synchronize()
    return a, h, s


@pytest.mark.parametrize("name,keep", PARAMS, ids=IDS)
def test_eager_and_async_match_the_oracle(name, keep):
    w = weights(name)
    verdict, a_ref, h_ref = oracle_verdict(w, keep, M, SEED)
    x = torch.from_numpy(w[None]).cuda()
    if verdict == OK:
        a, h = api.assign_hypotheses(x, M, SEED, maxExperts=keep)
        assert np.array_equal(a[0].cpu().numpy(), a_ref) and np.array_equal(h[0].cpu().numpy(), h_ref)
    else:
        with pytest.raises(RuntimeError, match=MESSAGES[verdict].replace("(", r"\(")):
            api.assign_hypotheses(x, M, SEED, maxExperts=keep)
    a, h, s = _async(x, M, SEED, maxExperts=keep)
    assert s.tolist() == [verdict]
    if verdict == OK:
        assert np.array_equal(a[0].cpu().numpy(), a_ref) and np.array_equal(h[0].cpu().numpy(), h_ref)


@pytest.mark.parametrize("w,keep", [([0.2, float("nan"), 0.1], 2), ([float("nan"), 0.1, 0.2, 0.3], 2),
                                    ([0.2, float("nan"), 0.1], 1), ([0.3, float("nan"), 0.2, float("nan"), 0.1], 2)])
def test_a_nan_under_the_clamp_is_refused(w, keep):
    """A NaN sorts above every number, so the clamp keeps it and the row is refused: the eager call raises torch's
    message and the stream-ordered one marks the row 1, in a batch whose other rows draw as usual."""
    w = np.array(w, np.float32)
    assert torch.isnan(torch_clamp(w, keep)).any()
    with pytest.raises(RuntimeError, match="inf, nan or element < 0"):
        api.assign_hypotheses(torch.from_numpy(w[None]).cuda(), M, SEED, maxExperts=keep)
    good = np.linspace(0.1, 0.9, len(w)).astype(np.float32)
    rows = torch.from_numpy(np.stack([good, w, good])).cuda()
    a, h, s = _async(rows, M, SEED, maxExperts=keep)
    assert s.tolist() == [OK, BAD_ENTRY, OK]
    a_ref, h_ref = O.assign_hypotheses(good[None], M, SEED, keep_top=keep)
    assert np.array_equal(a[0].cpu().numpy(), a_ref[0]) and np.array_equal(h[0].cpu().numpy(), h_ref[0])


@pytest.mark.parametrize("E,keep", [(10, 3), (64, 17), (1024, 50)])
def test_ties_resolve_as_the_stable_sort(E, keep):
    """Rows of repeated values: the experts kept are those torch.sort(stable=True) leaves on top, and the draw is the
    oracle's bit for bit."""
    rng = np.random.default_rng(E)
    rows = np.stack([np.full(E, 0.5, np.float32),                                  # all tied
                     rng.integers(1, 4, E).astype(np.float32) / 4,                 # three values, many ties each
                     np.where(rng.random(E) < 0.5, np.float32(0.25), np.float32(0.0)).astype(np.float32)])
    x = torch.from_numpy(rows).cuda()
    a, h = api.assign_hypotheses(x, 4096, SEED, maxExperts=keep)
    a_ref, h_ref = O.assign_hypotheses(rows, 4096, SEED, keep_top=keep)
    assert np.array_equal(a.cpu().numpy(), a_ref) and np.array_equal(h.cpu().numpy(), h_ref)
    for b in range(len(rows)):
        kept = (torch_clamp(rows[b], keep) > 0).numpy()
        drawn = h[b].cpu().numpy() > 0
        assert not (drawn & ~kept).any()
        if b == 0:
            assert np.nonzero(kept)[0].tolist() == list(range(E - keep, E)) and drawn[E - keep:].all()
    a2, h2, s2 = _async(x, 4096, SEED, maxExperts=keep)
    assert torch.equal(a2, a) and torch.equal(h2, h) and s2.tolist() == [OK] * len(rows)


def test_the_1024_expert_bound():
    """E = 1024 (the experts one CTA holds) with keep 50 and 4096 hypotheses; 1025 is refused by both calls."""
    rng = np.random.default_rng(7)
    w = (rng.random((3, 1024)) ** 8).astype(np.float32)
    w[1, ::3] = w[1, 0]                                                       # ties across the cut of the clamp
    w[2, 900:] = 1e-40                                                        # subnormal tail
    for keep in (50, -1):
        a_ref, h_ref = O.assign_hypotheses(w, 4096, SEED, keep_top=keep)
        x = torch.from_numpy(w).cuda()
        a, h = api.assign_hypotheses(x, 4096, SEED, maxExperts=keep)
        assert np.array_equal(a.cpu().numpy(), a_ref) and np.array_equal(h.cpu().numpy(), h_ref)
        a2, h2, s2 = _async(x, 4096, SEED, maxExperts=keep)
        assert torch.equal(a2, a) and torch.equal(h2, h) and s2.tolist() == [OK] * 3
    big = torch.rand(2, 1025, device="cuda")
    with pytest.raises(RuntimeError, match="E=1025 exceeds"):
        api.assign_hypotheses(big, 64, SEED)
    with pytest.raises(RuntimeError, match="E=1025 exceeds"):
        _async(big, 64, SEED)


@pytest.mark.parametrize("E", [1, 2, 19, 1024])
def test_histogram_is_torch_histc_of_the_draws(E):
    """e_hyps_hist = torch.histc(e_hyps.float(), bins=E, min=0, max=E-1), as the callers build it (train_esac.py:140)."""
    g = torch.Generator().manual_seed(E)
    probs = torch.softmax(3 * torch.randn(4, E, generator=g), dim=1).cuda()
    for kw in (dict(), dict(maxExperts=max(E // 3, 1)), dict(expertSelection=True)):
        a, h = api.assign_hypotheses(probs, 4096, SEED, **kw)
        for b in range(4):
            assert torch.equal(torch.histc(a[b].float(), bins=E, min=0, max=E - 1), h[b]), (b, kw)
        assert (h.sum(1) == 4096).all()


def _g_test_p(counts: np.ndarray, p: np.ndarray) -> float:
    """p-value of the G-test of `counts` against probabilities `p`, bins of expected count below 5 merged into one."""
    from scipy.stats import chi2
    expected = counts.sum() * p
    small = expected < 5
    obs = np.concatenate([counts[~small], [counts[small].sum()]]) if small.any() else counts
    exp = np.concatenate([expected[~small], [expected[small].sum()]]) if small.any() else expected
    keep = exp > 0
    assert (obs[~keep] == 0).all(), "drew an expert of probability 0"
    obs, exp = obs[keep], exp[keep]
    nz = obs > 0
    g = 2.0 * np.sum(obs[nz] * np.log(obs[nz] / exp[nz]))
    return float(chi2.sf(g, max(len(obs) - 1, 1)))


def _g_weights():
    rng = np.random.default_rng(11)
    peaky = rng.random(40) ** 8
    dominant = np.full(1000, 1e-6)
    dominant[123] = 1.0
    return {"peaky": (peaky, -1), "peaky_keep5": (peaky, 5), "uniform": (np.full(64, 0.5), -1),
            "dominant_and_1e-6": (dominant, -1), "subnormal_only": (rng.random(30) * 1e-39, -1),
            "ties_keep7": (np.repeat([0.1, 0.2, 0.3], 5), 7)}


@pytest.mark.parametrize("name", list(_g_weights()))
def test_counts_follow_the_clamped_distribution(name):
    """A test that does not share the oracle's algorithm: B = 64 rows of the same weights, 4096 draws each, the pooled
    counts against the float64 probabilities of the torch-clamped weights (G-test, bins of expected count < 5 merged,
    threshold 1e-6).  The draws are a pure function of the seed, so the outcome is fixed."""
    w, keep = _g_weights()[name]
    w = np.asarray(w, np.float32)
    clamped = torch_clamp(w, keep).double().numpy()
    p = clamped / clamped.sum()
    x = torch.from_numpy(np.tile(w, (64, 1))).cuda()
    a, h = api.assign_hypotheses(x, 4096, 77, maxExperts=keep)
    counts = h.double().sum(0).cpu().numpy()
    assert counts.sum() == 64 * 4096
    pv = _g_test_p(counts, p)
    assert pv > 1e-6, (name, pv)
