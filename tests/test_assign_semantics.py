"""The hypothesis assignment's semantics at its edges, on the CPU: oracle.esac_oracle.clamp_probs and assign_hypotheses
against the callers' own torch code -- util.clamp_probs (util.py:38-48) restated on torch.sort, then torch.multinomial's
error rules -- for NaN, +-inf, negatives, -0.0, subnormals and ties, with maxExperts 0, 1, E-1, E and E+5.

torch.sort (ascending) puts NaN after every number, so a NaN survives the keep-top clamp before any number does and
torch.multinomial then refuses the row.  CASES and keeps() are the fixture list of tests/test_gpu_assign_edges.py, which
holds the device kernel to the oracle on the same inputs."""
import numpy as np
import pytest
import torch

from oracle import esac_oracle as O

NAN, INF = float("nan"), float("inf")

CASES = {
    "nan_middle": [0.2, NAN, 0.1],
    "nan_first": [NAN, 0.1, 0.2, 0.3],
    "nan_last": [0.3, 0.1, 0.2, NAN],
    "two_nans": [0.3, NAN, 0.2, NAN, 0.1],
    "nan_and_inf": [INF, NAN, 0.5, 0.2],
    "pos_inf": [0.2, INF, 0.1, 0.3],
    "neg_inf": [0.2, -INF, 0.1, 0.3],
    "negative": [0.2, -1.0, 0.1, 0.4],
    "negative_smallest": [0.2, 0.3, -1e-30, 0.4, 0.1],
    "neg_zero": [-0.0, 0.3, -0.0, 0.1],
    "zeros_of_both_signs": [-0.0, 0.0, -0.0],
    "all_zero": [0.0, 0.0, 0.0, 0.0],
    "subnormal_only": [1e-40, 3e-45, 2e-39, 0.0, 1e-41],
    "subnormal_and_normal": [1e-40, 0.5, 1e-45, 0.25],
    "ties": [0.25, 0.25, 0.5, 0.25, 0.5, 0.25],
    "all_equal": [0.125] * 8,
    "single_positive": [0.0, 0.0, 0.7, 0.0, 0.0],
    "one_expert": [0.3],
    "peaky": (np.random.default_rng(5).random(19) ** 6).tolist(),
}


def weights(name: str) -> np.ndarray:
    return np.array(CASES[name], np.float32)


def keeps(E: int) -> list:
    """maxExperts values of a row of E experts: no clamp, 0, 1, E-1, E and E+5."""
    return sorted({-1, 0, 1, max(E - 1, 0), E, E + 5})


PARAMS = [(name, k) for name in CASES for k in keeps(len(CASES[name]))]
IDS = [f"{name}-keep{k}" for name, k in PARAMS]


def torch_clamp(w: np.ndarray, n: int) -> torch.Tensor:
    """util.clamp_probs, line for line on torch.sort (stable, so that ties resolve one way)."""
    probs = torch.from_numpy(np.array(w, np.float32))
    if n < 0:
        return probs
    s_prob, s_indx = probs.sort(dim=0, stable=True)
    for i, idx in enumerate(s_indx):
        if i < s_prob.size(0) - n:
            probs[idx] = 0
    return probs


# what torch.multinomial reports, as the status of the stream-ordered assignment numbers it
OK, BAD_ENTRY, ZERO_SUM = 0, 1, 2
MESSAGES = {BAD_ENTRY: "inf, nan or element < 0", ZERO_SUM: "sum of probabilities <= 0"}


def torch_verdict(probs: torch.Tensor) -> int:
    """torch.multinomial(probs, M, True) accepts the row (OK), refuses an entry (NaN, infinite or negative: BAD_ENTRY) or
    refuses the row's sum (ZERO_SUM).  The CPU and CUDA messages differ in wording, not in the rule."""
    try:
        torch.multinomial(probs, 16, True)
    except RuntimeError as e:
        msg = str(e)
        if "sum of probabilities" in msg:
            return ZERO_SUM
        if "< 0" in msg or "inf" in msg.lower() or "nan" in msg.lower():
            return BAD_ENTRY
        raise
    return OK


def oracle_verdict(w: np.ndarray, n: int, M: int = 64, seed: int = 3):
    """(verdict, assignment, histogram) of oracle.assign_hypotheses on one row; None, None on an error."""
    try:
        a, h = O.assign_hypotheses(w[None], M, seed=seed, keep_top=n)
    except RuntimeError as e:
        for v, msg in MESSAGES.items():
            if msg in str(e):
                return v, None, None
        raise
    return OK, a[0], h[0]


@pytest.mark.parametrize("name,keep", PARAMS, ids=IDS)
def test_clamp_keeps_what_the_torch_sort_keeps(name, keep):
    w = weights(name)
    ref = torch_clamp(w, keep).numpy()
    got = O.clamp_probs(w, keep)
    assert got.dtype == np.float32
    assert got.view(np.uint32).tolist() == ref.view(np.uint32).tolist(), (got, ref)   # bitwise: NaN and -0.0 included


@pytest.mark.parametrize("name,keep", PARAMS, ids=IDS)
def test_assignment_refuses_what_torch_multinomial_refuses(name, keep):
    w = weights(name)
    probs = torch_clamp(w, keep)
    want = torch_verdict(probs)
    got, a, h = oracle_verdict(w, keep)
    assert got == want, (got, want)
    if got == OK:
        pos = probs.numpy() > 0
        assert pos[a].all(), "drew an expert of zero probability"
        assert h.sum() == 64 and np.array_equal(h, np.bincount(a, minlength=len(w)).astype(np.float32))
        assert torch.equal(torch.histc(torch.from_numpy(a).float(), bins=len(w), min=0, max=len(w) - 1),
                           torch.from_numpy(h))


@pytest.mark.parametrize("w,keep", [([0.2, NAN, 0.1], 2), ([NAN, 0.1, 0.2, 0.3], 2), ([0.2, NAN, 0.1], 1),
                                    ([0.3, NAN, 0.2, NAN, 0.1], 2)])
def test_a_nan_survives_the_clamp_and_is_refused(w, keep):
    """The rows where ranking NaN below every number would zero the NaN and draw from the rest."""
    w = np.array(w, np.float32)
    probs = torch_clamp(w, keep)
    assert torch.isnan(probs).any()
    assert torch_verdict(probs) == BAD_ENTRY
    assert oracle_verdict(w, keep)[0] == BAD_ENTRY


def test_ties_resolve_as_the_stable_sort():
    """Among equal weights the later index sorts higher, so it keeps its place."""
    w = np.array([0.5] * 10, np.float32)
    assert np.nonzero(O.clamp_probs(w, 3))[0].tolist() == [7, 8, 9]
    w = np.array([0.25, 0.5, 0.25, 0.5, 0.25, 0.1], np.float32)
    assert np.nonzero(O.clamp_probs(w, 3))[0].tolist() == [1, 3, 4]
    assert np.nonzero(O.clamp_probs(np.array([-0.0, 0.0, 0.3, -0.0], np.float32), 2))[0].tolist() == [2]
