#!/usr/bin/env python
"""Fixed cost of a solver.run() call on the benchmark's workload, separated from the cost of an iteration.

    python tools/run_overhead.py [--tree DIR] [--reps 7] [--quick] [--out FILE]

On C2 (`bench.c2_edges(0)`, `bench.initial_iterate(0)`, as bench.py builds it), after a warm-up, `run(k)` windows for
k in 1, 5, 20, 100, 300 are timed between CUDA events exactly as bench.py times its windows (event, run(k), event,
synchronise); the k values alternate, `--reps` rounds.  A least-squares fit of the median window time,
t(k) = a + b k, gives a, the fixed cost of one call (launches, status reads, the device idling between rounds, surplus
steps), and b, the cost of one iteration.  bench.py's windows are run(20): a / 20 is the share of a in its step time.

Per window the tool also counts the steps the call enqueued (kernel launches but the call's resume kernel, over the
three kernels of a C2 step: head, vector, owner) against the closure evaluations it needed (func_evals before and after), and, where the library
reports it (mde_solver_debug_run_steps), the steps that ran: launched - ran are the surplus steps that exited at their
gates after the pause.

`--tree DIR` takes bench.py and pymde_b200 (with its built library) from another checkout, so that two builds can be
compared in one session.  Prints one JSON line (the card's name, power limit and SM clock cap read in the same
process) and writes it to `--out`.  `--quick` rehearses at a tiny size.  There is no CPU path: without a CUDA device
the tool stops with an error."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

KS = (1, 5, 20, 100, 300)
KERNELS_PER_STEP = 3  # C2 (Centered, m = 2): head, vector and owner kernels; the centring is fused into the vector pass
WARMUP = 10


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    sys.path.insert(0, tree)
    import torch
    import bench
    import pymde_b200 as pm
    from pymde_b200 import _lib
    assert os.path.dirname(os.path.abspath(pm.__file__)) == os.path.join(tree, "pymde_b200")
    lib = _lib.load()
    n = 3000 if args.quick else bench.N_ITEMS
    edges, w = bench.c2_edges(0, n=n) if args.quick else bench.c2_edges(0)
    X0 = bench.initial_iterate(0, n=n) if args.quick else bench.initial_iterate(0)
    if not torch.cuda.is_available():
        raise SystemExit("run_overhead: no CUDA device; nothing here is measured on the CPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, bench.EMBED_DIM, torch.tensor(edges, device=dev), f, pm.Centered(), device=dev)
    total = WARMUP + args.reps * sum(KS)
    solver = mde._solver(mde.constraint, 10, total + 8)
    solver.begin(torch.tensor(X0, device=dev), 0.0)
    solver.run(WARMUP)
    torch.cuda.synchronize()
    run_steps = getattr(lib, "mde_solver_debug_run_steps", None)  # (absent from builds before the progress word)

    done = WARMUP
    fe0 = solver.stats(done)[4]
    rows = {k: [] for k in KS}
    for rep in range(args.reps):
        for k in (KS if rep % 2 == 0 else KS[::-1]):
            l0 = int(lib.mde_launch_count())
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            d, _ = solver.run(k)
            ev1.record()
            torch.cuda.synchronize()
            us = ev0.elapsed_time(ev1) * 1e3
            launches = int(lib.mde_launch_count()) - l0
            assert d == done + k, (d, done, k)
            done = d
            fe = solver.stats(done)[4]
            row = {"us": us, "launched": (launches - 1) / KERNELS_PER_STEP, "evals": int(fe - fe0)}
            fe0 = fe
            if run_steps is not None:
                la, ran = C.c_int64(0), C.c_int64(0)
                _lib.check(run_steps(solver.handle, C.byref(la), C.byref(ran)))
                assert la.value * KERNELS_PER_STEP + 1 == launches, (la.value, launches)
                row["ran"] = int(ran.value)
            rows[k].append(row)

    med = {k: float(np.median([r["us"] for r in rows[k]])) for k in KS}
    b, a = np.polyfit(np.array(KS, dtype=np.float64), np.array([med[k] for k in KS]), 1)
    res = {"tree": tree, "gpu": bench.gpu_identity(dev), "n": n, "p": int(len(edges)), "reps": args.reps,
           "a_us_per_call": float(a), "b_us_per_iter": float(b),
           "window_us_median": {str(k): med[k] for k in KS},
           "us_per_iter": {str(k): med[k] / k for k in KS},
           "window_us_spread": {str(k): [float(min(r["us"] for r in rows[k])), float(max(r["us"] for r in rows[k]))]
                                for k in KS},
           "steps_launched_mean": {str(k): float(np.mean([r["launched"] for r in rows[k]])) for k in KS},
           "evals_mean": {str(k): float(np.mean([r["evals"] for r in rows[k]])) for k in KS}}
    if run_steps is not None:
        res["surplus_steps_max"] = {str(k): max(r["launched"] - r["ran"] for r in rows[k]) for k in KS}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
