"""The solver step computes fixed bits: sha1 digests of the embedding and of the statistics after 60 iterations,
recorded on an H100 from the build before the head kernel's history loads were reorganised
(tests/golden/solver_bits.json, written by tests/golden/make_solver_bits_golden.py).  Every history dot keeps its
thread, its elements, its FFMA chain, its warp tree and its fp64 order over blocks, so a change to how the head kernel
fetches the pairs or spreads them over blocks must reproduce these bits.

Cases: the C2 slice generator (n = 20 000, Centered m = 2) at memory 1, 4, 5, 6, 10, 11, 15, 16 and 32 (partial,
full and several 10-pair slices, and the boundaries of 5-pair ones); Centered m = 1 and 4; Standardized and Anchored
at m = 2; and a solve at n = 150 000, where the head pass is more than one wave of blocks (a grid-stride loop)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import bench

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "solver_bits.json")
ITERS = 60

CASES = (["c2slice-centered-m2-mem%d" % k for k in (1, 4, 5, 6, 10, 11, 15, 16, 32)] +
         ["c2slice-centered-m1-mem10", "c2slice-centered-m4-mem10", "c2slice-standardized-m2-mem10",
          "c2slice-anchored-m2-mem10", "large-centered-m2-mem15"])


@pytest.fixture(scope="module")
def recorded():
    with open(GOLDEN) as fh:
        return json.load(fh)


def _digest(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def evaluate(case):
    """{"x_sha1": ..., "stats_sha1": ...} of `case`: ITERS iterations of the device solver on the library as built."""
    import pymde_b200 as pm
    dev = torch.device("cuda", 0)
    kind, cname, mtag, memtag = case.split("-")
    m, memory = int(mtag[1:]), int(memtag[3:])
    n, k = (20000, 15) if kind == "c2slice" else (150000, 5)
    edges, w = bench.c2_edges(0, n=n, k=k)
    X0 = bench.initial_iterate(1, n=n, m=m)
    if cname == "centered":
        cons = pm.Centered()
    elif cname == "standardized":
        cons = pm.Standardized()
    else:
        anchors = np.arange(0, n, n // 9)[:9]
        values = np.random.default_rng(5).standard_normal((len(anchors), m)).astype(np.float32)
        cons = pm.Anchored(torch.tensor(anchors, device=dev), torch.tensor(values, device=dev))
        X0[anchors] = values
    f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, m, torch.tensor(edges, device=dev), f, cons, device=dev)
    if cname == "standardized":
        X0 = cons.project_onto_constraint(torch.tensor(X0, device=dev)).cpu().numpy()
    solver = mde._solver(mde.constraint, memory, ITERS + 1)
    solver.begin(torch.tensor(X0, device=dev), 0.0, ITERS + 1)
    done, _ = solver.run(ITERS)
    assert done == ITERS
    avg, res, pct, stp, fe = solver.stats(ITERS)
    X = solver.x_view().cpu().numpy()
    assert np.isfinite(X).all()
    stats = [np.asarray(a, dtype=np.float64) for a in (avg, res, pct, stp)] + [np.asarray(fe, dtype=np.int64)]
    return {"x_sha1": _digest(X), "stats_sha1": _digest(*stats)}


def test_fixture_lists_every_case(recorded):
    assert sorted(recorded["cases"]) == sorted(CASES)
    assert "H100" in recorded["gpu"]


@gpu
@pytest.mark.parametrize("case", CASES)
def test_solver_reproduces_the_recorded_bits(case, recorded):
    assert evaluate(case) == recorded["cases"][case]
