"""CPU: the fp64 replay of tests/lbfgs_replay.py accepts the fp32 oracle's own solves at memory 1, 3, 10, 11 and 32 (each
past at least one full wrap of the history), one whose every pair is rejected and one that resets its history 50
times, and it rejects readouts of a solver
with each of six faults: the newest pair evicted instead of the oldest, the direction formed with pair j - 10 in
place of pair j (a slice-offset error of the device's 10-pair slices), H_diag from the oldest pair, the centering
skipped for one iteration, g_prev lagging one iteration, and the history thrown away (a reset) after a step that
was not 0.  Each faulty readout is what that solver would report at
the first pause the fault touches, its direction recomputed from its own (faulty) state, so only the rule the fault
breaks can catch it."""
import copy

import numpy as np
import pytest

from oracle import mde_oracle as O
from tests import lbfgs_replay as L

N_ROWS = 300


def _case(memory, scale=1.0, iters=None):
    edges, w = L.knn_graph(N_ROWS, 6, 11, scale)
    cons = O.Centered()
    prob = L.Problem(edges, L.push_pull_spec(w), cons)
    X0 = L.initial_point(N_ROWS, 2, cons, 3)
    pauses, stats = L.oracle_trace(prob, X0, memory, iters or 2 * memory + 12)
    return prob, pauses, stats


@pytest.fixture(scope="module")
def traces():
    return {}


def _trace(traces, memory, scale=1.0):
    if (memory, scale) not in traces:
        traces[(memory, scale)] = _case(memory, scale)
    return traces[(memory, scale)]


@pytest.mark.parametrize("memory", [1, 3, 10, 11, 32])
def test_replay_accepts_the_fp32_oracle(traces, memory):
    prob, pauses, stats = _trace(traces, memory)
    R = L.replay(pauses, stats, prob, memory)
    assert R.evicted >= memory + 1, "the trace must wrap the history at least once"
    assert R.accepted + R.rejected == len(pauses) - 2


def test_replay_accepts_rejected_pairs():
    """Weights scaled by 1e-4: y.s < 1e-10 from the first pair on, so every pair is rejected, the history stays
    empty and d = -g_prev with H_diag = 1 at every pause."""
    prob, pauses, stats = _case(3, scale=1e-4, iters=20)
    R = L.replay(pauses, stats, prob, 3)
    assert R.accepted == 0 and R.rejected == len(pauses) - 2
    assert all(p["count"] == 0 and p["H_diag"] == 1.0 for p in pauses[1:])


def test_replay_follows_resets(golden):
    """docs5 (Quadratic, Standardized, n = 5) for 60 iterations at eps = 0: once it has converged its line searches
    end at t = 0 and every iteration resets the history (optim.py:172-173); the oracle's trace resets 50 times."""
    g = golden["trajectories"]
    prob = L.Problem(g["docs5/edges"], O.FnSpec(O.P_QUADRATIC, g["docs5/par0"]), O.Standardized())
    pauses, stats = L.oracle_trace(prob, g["docs5/X0"], 10, 60)
    R = L.replay(pauses, stats, prob, 10)
    assert R.resets >= 40


def _redirect(p):
    """Recompute the direction of a readout from its own g_prev, pairs and H_diag (a solver consistent with its
    state)."""
    p["d"] = L.explicit_two_loop(p["g_prev"].reshape(-1).astype(np.float64),
                                 [v.reshape(-1).astype(np.float64) for v in p["S"]],
                                 [v.reshape(-1).astype(np.float64) for v in p["Y"]],
                                 p["H_diag"]).astype(np.float32).reshape(p["g_prev"].shape)


def _first(pauses, pred):
    return next(k for k in range(2, len(pauses)) if pred(pauses[k - 1], pauses[k]))


def _evict_newest(pauses, stats, memory):
    k = _first(pauses, lambda P, Q: P["count"] == memory and Q["count"] == memory)
    Q = pauses[k]
    P = pauses[k - 1]
    Q["S"] = np.concatenate([P["S"][:-1], Q["S"][-1:]])
    Q["Y"] = np.concatenate([P["Y"][:-1], Q["Y"][-1:]])
    _redirect(Q)


def _slice_offset(pauses, stats, memory):
    k = _first(pauses, lambda P, Q: Q["count"] > 10)
    Q = pauses[k]
    idx = [j - 10 if j >= 10 else j for j in range(Q["count"])]
    held = Q["S"], Q["Y"]
    Q["S"], Q["Y"] = Q["S"][idx], Q["Y"][idx]
    _redirect(Q)
    Q["S"], Q["Y"] = held  # the history itself is intact: only the direction read the wrong pairs


def _h_from_oldest(pauses, stats, memory):
    k = _first(pauses, lambda P, Q: Q["count"] >= 2)
    Q = pauses[k]
    s, y = Q["S"][0].reshape(-1).astype(np.float64), Q["Y"][0].reshape(-1).astype(np.float64)
    Q["H_diag"] = float(np.float32(y @ s) / np.float32(y @ y))
    _redirect(Q)


def _skip_centering(pauses, stats, memory):
    # iteration 0 starts off centre: its retraction is the one whose mean matters
    P, Q = pauses[0], pauses[1]
    Q["X"] = (P["X"] + np.float32(stats["steplen"][0]) * Q["d"]).astype(np.float32)


def _lagging_g_prev(pauses, stats, memory):
    k = _first(pauses, lambda P, Q: Q["n_iter"] >= 3)
    pauses[k]["g_prev"] = pauses[k - 1]["g_prev"].copy()
    _redirect(pauses[k])


def _spurious_reset(pauses, stats, memory):
    k = _first(pauses, lambda P, Q: Q["count"] >= 3)
    Q = pauses[k]
    Q["n_iter"], Q["count"], Q["H_diag"] = 0, 0, 1.0
    Q["S"], Q["Y"] = Q["S"][:0], Q["Y"][:0]


FAULTS = {
    "evict_newest": (_evict_newest, "not appended"),
    "slice_offset": (_slice_offset, "direction"),
    "h_from_oldest": (_h_from_oldest, "h_diag"),
    "skip_centering": (_skip_centering, "move"),
    "lagging_g_prev": (_lagging_g_prev, "g_prev is not"),
    "spurious_reset": (_spurious_reset, "n_iter 0 after"),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_replay_rejects_injected_faults(traces, fault):
    memory = 11
    prob, pauses, stats = _trace(traces, memory)
    bad = copy.deepcopy(pauses)
    inject, message = FAULTS[fault]
    inject(bad, stats, memory)
    with pytest.raises(AssertionError, match=message):
        L.replay(bad, stats, prob, memory)
