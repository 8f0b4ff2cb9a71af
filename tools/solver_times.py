"""Where a solver step spends its time: %globaltimer stamps of the head kernel's scalar stage (see
mde_solver_debug_times in include/mde_b200.h) on the C2-shaped bench problem, sampled after runs of different length."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bench
import pymde_b200 as pm

dev = torch.device("cuda", 0)
edges, w = bench.c2_edges(0)
X0 = torch.tensor(bench.initial_iterate(0), device=dev)
f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
mde = pm.MDE(bench.N_ITEMS, bench.EMBED_DIM, torch.tensor(edges, device=dev), f, pm.Centered(), device=dev)
solver = mde._solver(mde.constraint, 10, 400)
names = ["pass(last block)", "stage state", "reduce", "finish prev", "direction", "colsums", "writeback+exit->vec"]
acc = []
for iters in (30, 31, 33, 37, 45, 60, 80):
    solver.begin(X0, 0.0, iters)
    solver.run(iters)
    out = (C.c_ulonglong * 8)()
    solver.lib.mde_solver_debug_times(solver.handle, out, None)
    t = np.array(list(out), dtype=np.float64)
    acc.append(np.diff(t) / 1000.0)
    print(iters, " ".join("%s=%.2f" % (n, d) for n, d in zip(names, acc[-1])), "total=%.2f us" % ((t[7] - t[0]) / 1000.0))
print("median", " ".join("%s=%.2f" % (n, d) for n, d in zip(names, np.median(np.array(acc), 0))))
