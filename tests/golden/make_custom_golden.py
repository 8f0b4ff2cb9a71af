"""Generate tests/golden/custom_constraints.npz by RUNNING THE UNMODIFIED REFERENCE (cvxgrp/pymde v0.2.1) on a
user-defined constraint: the reference's own `_Sphere(1.0)` (pymde/constraints.py:203-231, rows of X on the unit
sphere), which no built-in constraint of the device solver covers.

Run with the reference importable (oracle/ref_loader.py), on the CPU:

    PYMDE_REFERENCE=<reference checkout with its Cython extension built> python tests/golden/make_custom_golden.py

Case `sphere`: n = 400, m = 3, PushAndPull(Log1p, Log) on make_golden.py's k-NN-like ring graph (weights 1 or 2)
plus as many random repulsive pairs (weight -1), fp32, 60 iterations from `_Sphere(1.0).initialization` under
torch.manual_seed(0).  Stored: X0, edges, par0 (the weights), the statistics and the final value of the solve with
one torch thread, and the statistics and final value of the same solve with 4 threads (`t4/...`): the fp32
summation order of the reference depends on the thread count, so the two runs record its own spread.  For the
Anchored constraint the tests use anchored.npz (make_golden.py)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import knn_like_graph, pymde  # noqa: E402  (loads the reference, 1 torch thread)


def gen_sphere():
    out = {}
    pen = pymde.penalties
    rng = np.random.default_rng(31)
    n, m, iters = 400, 3, 60
    att = knn_like_graph(n, 4, rng)
    attset = set(map(tuple, att))
    rep = []
    while len(rep) < len(att):
        i, j = rng.integers(0, n, 2)
        if i != j and (min(i, j), max(i, j)) not in attset:
            rep.append((min(i, j), max(i, j)))
            attset.add((min(i, j), max(i, j)))
    edges = np.concatenate([att, np.array(rep, dtype=np.int64)])
    w = np.concatenate([rng.choice([1.0, 2.0], len(att)), -np.ones(len(rep))]).astype(np.float32)
    cons = pymde.constraints._Sphere(1.0)
    torch.manual_seed(0)
    X0 = cons.initialization(n, m)
    out["sphere/X0"], out["sphere/edges"], out["sphere/par0"] = X0.numpy().copy(), edges, w
    out["sphere/max_iter"] = np.array(iters)
    for th, tag in ((1, "sphere"), (4, "sphere/t4")):
        torch.set_num_threads(th)
        f = pen.PushAndPull(torch.tensor(w), pen.Log1p, pen.Log)
        mde = pymde.MDE(n, m, torch.tensor(edges), f, cons)
        X = mde.embed(X=X0.clone(), max_iter=iters, eps=1e-5)
        st = mde.solve_stats
        out[tag + "/average_distortions"] = np.array(st.average_distortions)
        out[tag + "/residual_norms"] = np.array(st.residual_norms)
        out[tag + "/step_size_percents"] = np.array(st.step_size_percents)
        out[tag + "/final_value"] = mde.average_distortion(X.detach()).numpy()
        if th == 1:
            out["sphere/X"] = X.detach().numpy().copy()
        print("sphere threads", th, "iters", st.iterations, "final", float(out[tag + "/final_value"]),
              "max | |x| - 1 |", float((X.norm(dim=1) - 1).abs().max()))
    torch.set_num_threads(1)
    np.savez_compressed(os.path.join(HERE, "custom_constraints.npz"), **out)
    print("custom_constraints.npz", len(out))


if __name__ == "__main__":
    gen_sphere()
