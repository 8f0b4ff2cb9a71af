#!/usr/bin/env python
"""Milliseconds per embed() iteration on the C2 problem (bench.py's workload, built with bench.py's own
generators, PushAndPull(Log1p, Log) as the table function) for user-defined constraints:

  centered  a user-written clone of Centered (Z -= Z.mean(0)); baseline arm: the built-in Centered()
  sphere    rows on the unit sphere (the reference's _Sphere(1.0)), from the normalised C2 start

each in three arms: graph (PYMDE_B200_CONSTRAINT=graph: projections captured into the device solver's step
graphs), hook (=hook: called back at every step) and generic (unset: the host-stepped solver).  Each arm: one warm-up
embed(), then `--repeats` timed embed(X0, max_iter=K, eps=0) calls bracketed by CUDA events and a synchronize; the
table reports the median over those windows of ms / iteration (capture and solver set-up included, amortised over K)
and the evaluations per iteration.  L2 is not flushed (warm-L2 numbers, as tools/external_times.py).  For the device
arms, the library's launch counter over 20 further iterations gives the solver's own kernels per iteration (steps
launched, surplus steps included, times kernels per step; the kernels of the user's torch code are not counted).

    python tools/constraint_times.py [--iters K] [--generic-iters K] [--repeats R] [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from external_times import time_embed  # noqa: E402


def constraints(torch, pm):
    Base = pm.constraints.Constraint

    class UserCentered(Base):
        def name(self):
            return "user-centered"

        def initialization(self, n_items, embedding_dim, device=None):
            X = torch.randn((int(n_items), int(embedding_dim)), device=device)
            return X - X.mean(0)

        def project_onto_constraint(self, Z, inplace=True):
            return Z.sub_(Z.mean(0)) if inplace else Z - Z.mean(0)

        def project_onto_tangent_space(self, X, Z, inplace=True):
            return Z

    class Sphere(Base):
        def name(self):
            return "sphere"

        def initialization(self, n_items, embedding_dim, device=None):
            X = torch.randn((int(n_items), int(embedding_dim)), device=device)
            return X / X.norm(dim=1)[:, None]

        def project_onto_constraint(self, Z, inplace=True):
            return Z.div_(Z.norm(dim=1)[:, None]) if inplace else Z / Z.norm(dim=1)[:, None]

        def project_onto_tangent_space(self, X, Z, inplace=True):
            dual = (Z * X).sum(1)
            return Z.sub_(dual[:, None] * X) if inplace else Z - dual[:, None] * X

    return UserCentered, Sphere


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
    from pymde_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("constraint_times.py measures on a CUDA device; none found")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    edges, w = bench.c2_edges(0)
    X0 = torch.tensor(bench.initial_iterate(0), device=dev)
    E = torch.tensor(edges, device=dev)
    wt = torch.tensor(w, device=dev)
    f = pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log)
    UserCentered, Sphere = constraints(torch, pm)
    starts = {"centered": X0 - X0.mean(0), "sphere": X0 / X0.norm(dim=1)[:, None]}
    result = {"gpu": bench.gpu_identity(dev), "workload": "C2: n=%d, m=%d, p=%d, PushAndPull(Log1p, Log)" % (
        bench.N_ITEMS, bench.EMBED_DIM, len(edges)), "l2": "warm (no flush between iterations)", "arms": {}}
    lib = _lib.load()

    arms = [("centered/builtin", pm.Centered, None, args.iters)]
    for cname, cls in (("centered", UserCentered), ("sphere", Sphere)):
        arms += [(cname + "/graph", cls, "graph", args.iters), (cname + "/hook", cls, "hook", args.iters),
                 (cname + "/generic", cls, "generic", args.generic_iters)]
    for name, make, mode, iters in arms:
        os.environ["PYMDE_B200_CONSTRAINT"] = mode or "generic"
        mde = pm.MDE(bench.N_ITEMS, bench.EMBED_DIM, E, f, make(), device=dev)
        start = starts[name.split("/")[0]]
        r = time_embed(torch, mde, start, iters, args.repeats)
        cur = mde.__dict__["_device_solver"]
        r["solver"] = "generic" if cur is None else (cur[1].constraint_mode or "builtin")
        if cur is not None:  # launches of one more solver run / the steps it took = kernels per step
            solver = cur[1]
            solver.begin(start, 0.0, 20)
            l0 = int(lib.mde_launch_count())
            solver.run(20)
            r["launches_per_iter_20"] = (int(lib.mde_launch_count()) - l0) / 20.0
        result["arms"][name] = r
        print("%-18s %9.4f ms/iter of embed()  %9s ms/iter of the solver alone  %5.2f evals/iter  %6s launches/iter "
              "(%s, %d iterations per embed)" % (
                  name, r["ms_per_iter"], "%.4f" % r["solver_ms_per_iter"] if "solver_ms_per_iter" in r else "-",
                  r["evals_per_iter"], "%.1f" % r["launches_per_iter_20"] if "launches_per_iter_20" in r else "-",
                  r["solver"], r["iterations"]), flush=True)
        del mde
    os.environ.pop("PYMDE_B200_CONSTRAINT", None)
    print("gpu: %s" % json.dumps(result["gpu"]))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
