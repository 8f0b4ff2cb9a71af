"""CPU: the policy by which mde_solver_run keeps the step queue fed from the device's progress word
(feed_policy in pymde_b200/csrc/mde_solver.cu, through its host-side debug entry point), run against a model of the
device: a step's head kernel ends at most one iteration, and the pause comes in the head that ends the last one.
No GPU compute involved."""
import numpy as np
import pytest

from pymde_b200 import _lib

BIG = 8  # steps of the multi-step graph


@pytest.fixture(scope="module")
def policy():
    lib = _lib.load()
    return lambda in_flight, left: int(lib.mde_dbg_feed_policy(in_flight, left))


def test_policy_table(policy):
    assert policy(0, 20) == BIG and policy(8, 20) == BIG  # two eight-step graphs ahead
    assert policy(9, 40) == 0 and policy(16, 40) == 0
    assert policy(0, 7) == 1 and policy(6, 7) == 1 and policy(7, 7) == 0  # near the pause: single steps, up to `left`
    assert policy(9, 12) == 0 and policy(7, 12) == 1
    assert policy(0, 0) == 1 and policy(1, 0) == 0 and policy(1, 1) == 0  # an empty queue always gets one step


def simulate(policy, costs, rng, max_lag):
    """One run() of len(costs) iterations, iteration i taking costs[i] evaluation steps.  The host reads a snapshot
    of the progress word up to `max_lag` heads old (the freshest one when the device would otherwise wait) and
    enqueues what the policy asks for; returns (steps launched, steps run, graph launches, device waits)."""
    target = len(costs)
    ends = 1 + np.cumsum(costs)        # head that ends iteration i (the first head of a resumed run starts one)
    stop = int(ends[-1])               # ... and the last of them pauses the solve
    launched = graphs = waits = 0
    j = 0                              # heads run
    while True:
        lag = int(rng.integers(0, max_lag + 1)) if max_lag else 0
        for fresh in (False, True):
            seen = j if fresh else max(0, j - lag)
            if seen >= stop:
                break
            while True:
                k = policy(launched - seen, target - int(np.searchsorted(ends, seen, side="right")))
                if not k:
                    break
                launched += k
                graphs += 1
            if launched > j:
                break
            waits += 1
        if j >= stop:
            return launched, j, graphs, waits
        assert launched > j, "the queue ran dry before the pause"
        j += 1


@pytest.mark.parametrize("target", [1, 2, 7, 8, 9, 20, 97, 300])
@pytest.mark.parametrize("max_lag", [0, 3])
def test_queue_stays_fed_and_no_step_is_enqueued_after_the_pause(policy, target, max_lag):
    rng = np.random.default_rng(target * 10 + max_lag)
    for trial in range(20):
        costs = np.ones(target, dtype=np.int64) if trial == 0 else rng.choice([1, 1, 1, 2, 3, 10], target)
        launched, ran, graphs, waits = simulate(policy, costs, rng, max_lag)
        assert ran == 1 + costs.sum()
        assert launched == ran, (launched, ran)
        if max_lag == 0:
            assert waits == 0
        if trial == 0 and target >= 20:
            # mostly eight-step graphs: one graph launch per ~8 steps, a few single steps near the pause
            assert graphs <= (target + 1) // BIG + BIG + 2, graphs
