"""A/B timing of MDE_B200_STEPS (steps per solver graph launch) on the bench workload (C2) and the
Standardized variant.  Not the headline bench (bench.py is)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bench, pymde_b200 as pm

dev = torch.device("cuda", 0)
edges, w = bench.c2_edges(0)
X0 = torch.tensor(bench.initial_iterate(0), device=dev)
et = torch.tensor(edges, device=dev)
wt = torch.tensor(w, device=dev)
ITERS = int(os.environ.get("VARIANT_ITERS", "400"))


def run(cons, env):
    os.environ.pop("MDE_B200_STEPS", None)
    os.environ.update(env)
    f = pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(bench.N_ITEMS, 2, et, f, cons, device=dev)
    Xs = X0.clone() if cons is pm.Centered() else pm.util.proj_standardized(X0.clone(), demean=True)
    solver = mde._solver(cons, 10, ITERS + 16)
    best = 0.0
    for rep in range(3):
        solver.begin(Xs, 0.0); solver.run(16); torch.cuda.synchronize()
        t0 = time.perf_counter(); done, _ = solver.run(ITERS); torch.cuda.synchronize(); dt = time.perf_counter() - t0
        best = max(best, (done - 16) / dt)
    avg, res, pct, stp, fe = solver.stats(done)
    return best, fe / done, avg[0], avg[-1], done


VARIANTS = [{}, {"MDE_B200_STEPS": "16"}, {"MDE_B200_STEPS": "32"}, {}]
for cname, cons in (("centered", pm.Centered()), ("standardized", pm.Standardized())):
    for env in VARIANTS:
        tag = " ".join("%s=%s" % (k.replace("MDE_B200_", ""), v) for k, v in sorted(env.items())) or "STEPS=8"
        try:
            r = run(cons, env)
            print("%-13s %-12s %8.0f it/s  evals/iter %.2f  loss %.6f -> %.6f  (%d iterations)" % ((cname, tag) + r), flush=True)
        except Exception as ex:
            print("%-13s %-12s FAILED: %s" % (cname, tag, ex), flush=True)
