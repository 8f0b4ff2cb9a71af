#!/usr/bin/env python
"""Milliseconds per embed() iteration on the C2 problem (bench.py's workload, built with bench.py's own
generators) for a distortion function given four ways:

  builtin  penalties.PushAndPull(w, Log1p, Log): the table function, fused kernels on the device solver
  graph    the same function as a torch callable, captured into the device solver's step graphs
  hook     the same callable, called back from the device solver at every evaluation
  generic  the same callable on the host-stepped solver (PYMDE_B200_EXTERNAL=generic)

Each arm: one warm-up embed(), then `--repeats` timed embed(X0, max_iter=K, eps=0) calls, each bracketed by CUDA
events on the launching stream and a synchronize; the table reports the median over those windows of
ms / iteration (capture and solver set-up included, amortised over K).  Nothing flushes the L2 between iterations:
C2's step working set (X, gradient, history, edge layout: ~40 MB) stays in the 50 MB L2, so the numbers are warm-L2
numbers.  The device arms are also timed as bench.py times its solver (begin, 5 warm-up iterations, then
mde_solver_run windows: no capture or step-graph build inside).  The torch part alone (the captured graph replayed
by itself, and eagerly) is timed too, with the evaluations per iteration, to show what graph mode is bound by.

    python tools/external_times.py [--iters K] [--generic-iters K] [--repeats R] [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def torch_push_and_pull(torch, wt):
    pos = wt >= 0

    def f(d):
        return torch.where(pos, wt * torch.log1p(d.pow(1.5)), wt * torch.log(-torch.expm1(-d)))

    return f


def time_embed(torch, mde, X0, iters, repeats):
    mde.embed(X=X0.clone(), max_iter=iters, eps=0.0)  # warm-up: module loads, capture, solver graphs
    out = []
    for _ in range(repeats):
        X = X0.clone()
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        mde.embed(X=X, max_iter=iters, eps=0.0)
        ev1.record()
        torch.cuda.synchronize()
        out.append(ev0.elapsed_time(ev1) / mde.solve_stats.iterations)
    st = mde.solve_stats
    r = {"ms_per_iter": float(np.median(out)), "windows_ms_per_iter": [round(v, 4) for v in out],
         "iterations": st.iterations, "evals_per_iter": st.func_evals / st.iterations,
         "final_distortion": float(st.average_distortions[-1])}
    cur = mde.__dict__["_device_solver"]
    if cur is not None:  # the device solver alone, as bench.py times it: no capture or graph build in the windows
        solver, steady = cur[1], []
        solver.begin(X0, 0.0, iters)
        solver.run(5)
        for _ in range(repeats):
            k = (iters - 5) // repeats
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            solver.run(k)
            ev1.record()
            torch.cuda.synchronize()
            steady.append(ev0.elapsed_time(ev1) / k)
        r["solver_ms_per_iter"] = float(np.median(steady))
    return r


def time_part(torch, part, reps=200):
    """ms per evaluation of the callable's torch part alone: its captured graph replayed, and the eager ops."""
    res = {}
    for name, fn in (("graph_replay", part.graph.replay), ("eager", part.run)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(reps):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        res[name + "_ms"] = ev0.elapsed_time(ev1) / reps
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=200, help="iterations per timed embed() (device arms)")
    ap.add_argument("--generic-iters", type=int, default=20, help="iterations per timed embed() (generic arm)")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    args = ap.parse_args()

    import torch
    import bench
    import pymde_b200 as pm
    from pymde_b200 import external

    if not torch.cuda.is_available():
        raise SystemExit("external_times.py measures on a CUDA device; none found")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    edges, w = bench.c2_edges(0)
    X0 = torch.tensor(bench.initial_iterate(0), device=dev)
    E = torch.tensor(edges, device=dev)
    wt = torch.tensor(w, device=dev)
    result = {"gpu": bench.gpu_identity(dev), "workload": "C2: n=%d, m=%d, p=%d, Centered" % (
        bench.N_ITEMS, bench.EMBED_DIM, len(edges)), "l2": "warm (no flush between iterations)", "arms": {}}

    arms = [("builtin", None, args.iters), ("graph", "graph", args.iters), ("hook", "hook", args.iters),
            ("generic", "generic", args.generic_iters)]
    for name, mode, iters in arms:
        if mode is None:
            os.environ.pop("PYMDE_B200_EXTERNAL", None)
            f = pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log)
        else:
            os.environ["PYMDE_B200_EXTERNAL"] = mode
            f = torch_push_and_pull(torch, wt)
        mde = pm.MDE(bench.N_ITEMS, bench.EMBED_DIM, E, f, pm.Centered(), device=dev)
        r = time_embed(torch, mde, X0, iters, args.repeats)
        cur = mde.__dict__["_device_solver"]
        r["solver"] = "generic" if cur is None else (cur[1].external_mode or "table")
        result["arms"][name] = r
        print("%-8s %9.4f ms/iter of embed()  %9s ms/iter of the solver alone  %5.2f evals/iter  (%s, %d iterations "
              "per embed)" % (name, r["ms_per_iter"], "%.4f" % r["solver_ms_per_iter"] if "solver_ms_per_iter" in r
                              else "-", r["evals_per_iter"], r["solver"], r["iterations"]), flush=True)
        del mde
    os.environ["PYMDE_B200_EXTERNAL"] = "graph"
    part = external.UserPart(torch_push_and_pull(torch, wt), len(edges), dev)
    result["torch_part"] = time_part(torch, part)
    os.environ.pop("PYMDE_B200_EXTERNAL", None)
    print("torch part alone: %.4f ms per evaluation as a graph, %.4f ms eager" % (
        result["torch_part"]["graph_replay_ms"], result["torch_part"]["eager_ms"]))
    print("gpu: %s" % json.dumps(result["gpu"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
