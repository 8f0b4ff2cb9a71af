"""Generate golden fixtures by RUNNING THE UNMODIFIED REFERENCE (cvxgrp/pymde v0.2.1).

Run with the reference importable (oracle/ref_loader.py):

    PYMDE_REFERENCE=<reference checkout with its Cython extension built> python tests/golden/make_golden.py

Outputs (committed): tests/golden/functions.npz, evals.npz, projections.npz,
trajectories.npz.  Tests read these files; none of them needs the reference.
Every array is produced by reference code paths only:
  functions    f(d) and autograd df/dd   pymde/functions/{penalties,losses}.py
  evals        MDE.average_distortion + backward   pymde/average_distortion.py:36-80
  projections  constraints + util.proj_standardized  pymde/constraints.py, pymde/util.py:129-171
  trajectories MDE.embed                 pymde/problem.py:386 -> pymde/optim.py:69 -> pymde/lbfgs.py
"""
import functools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
from oracle.ref_loader import load_reference  # noqa: E402

pymde = load_reference()
assert pymde is not None, "reference not importable"
torch.set_num_threads(1)  # bit-reproducible summation order (SURVEY Appendix C.4)


def function_cases(p, dtype, rng):
    """name -> (constructor kwargs as arrays, callable building the reference module)."""
    pen, los = pymde.penalties, pymde.losses
    w = torch.tensor(rng.uniform(0.2, 2.0, p), dtype=dtype)
    wneg = -w
    wmix = torch.tensor(rng.choice([1.0, 2.0, -1.0], p), dtype=dtype)
    dev = torch.tensor(rng.uniform(0.1, 3.0, p), dtype=dtype)
    w2 = torch.tensor(rng.uniform(0.2, 2.0, p), dtype=dtype)
    return {
        "pen_linear": (pen.Linear(w), dict(par0=w)),
        "pen_quadratic": (pen.Quadratic(w), dict(par0=w)),
        "pen_cubic": (pen.Cubic(w), dict(par0=w)),
        "pen_power_2.5": (pen.Power(w, 2.5), dict(par0=w)),
        "pen_huber_0.5": (pen.Huber(w, 0.5), dict(par0=w)),
        "pen_logistic_0.3_3": (pen.Logistic(w, 0.3, 3.0), dict(par0=w)),
        "pen_log1p_1.5": (pen.Log1p(w, 1.5), dict(par0=w)),
        "pen_log_1": (pen.Log(wneg, 1.0), dict(par0=wneg)),
        "pen_invpower_1": (pen.InvPower(wneg, 1), dict(par0=wneg)),
        "pen_logratio_2": (pen.LogRatio(wneg, 2), dict(par0=wneg)),
        "pen_pushpull_log1p_log": (pen.PushAndPull(wmix, pen.Log1p, pen.Log), dict(par0=wmix)),
        "pen_pushpull_default": (pen.PushAndPull(wmix), dict(par0=wmix)),
        "pen_pushpull_quad_invpower": (
            pen.PushAndPull(wmix, pen.Quadratic, pen.InvPower), dict(par0=wmix)),
        "loss_absolute": (los.Absolute(dev), dict(par0=dev)),
        "loss_quadratic": (los.Quadratic(dev), dict(par0=dev)),
        "loss_weighted_quadratic": (los.WeightedQuadratic(dev), dict(par0=dev)),
        "loss_weighted_quadratic_w": (los.WeightedQuadratic(dev, w2), dict(par0=dev, par1=w2)),
        "loss_huber_0.7": (los.Huber(dev, 0.7), dict(par0=dev)),
        "loss_cubic": (los.Cubic(dev), dict(par0=dev)),
        "loss_power_1.5": (los.Power(dev, 1.5), dict(par0=dev)),
        "loss_logistic": (los.Logistic(dev), dict(par0=dev)),
        "loss_fractional": (los.Fractional(dev), dict(par0=dev)),
        "loss_soft_fractional_10": (los.SoftFractional(dev, 10.0), dict(par0=dev)),
    }


def gen_functions():
    out = {}
    p = 64
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        rng = np.random.default_rng(7)
        cases = function_cases(p, dtype, rng)
        d = torch.tensor(rng.uniform(0.05, 4.0, p), dtype=dtype)
        for name, (f, pars) in cases.items():
            dd = d.clone().requires_grad_(True)
            val = f(dd)
            val.sum().backward()
            out["%s/%s/d" % (name, tag)] = d.numpy()
            out["%s/%s/f" % (name, tag)] = val.detach().numpy()
            out["%s/%s/fp" % (name, tag)] = dd.grad.numpy()
            for k, v in pars.items():
                out["%s/%s/%s" % (name, tag, k)] = v.numpy()
    np.savez_compressed(os.path.join(HERE, "functions.npz"), **out)
    print("functions.npz", len(out))


def random_graph(n, p, rng):
    pairs = set()
    while len(pairs) < p:
        i, j = rng.integers(0, n, 2)
        if i != j:
            pairs.add((min(i, j), max(i, j)))
    e = np.array(sorted(pairs), dtype=np.int64)
    rng.shuffle(e)
    return e


def gen_evals():
    out = {}
    rng = np.random.default_rng(11)
    for m, zero in ((1, False), (2, False), (3, False), (4, False), (7, False), (16, False),
                    (2, True), (3, True)):
        n, p = 60, 64
        edges = random_graph(n, p, rng)
        # flip some edges so i > j also occurs (tolerated, problem.py:80-83)
        flip = rng.random(p) < 0.3
        edges[flip] = edges[flip][:, ::-1]
        X = rng.standard_normal((n, m)).astype(np.float32)
        key = "m%d" % m
        if zero:  # a zero-distance pair is legal input (average_distortion.py:55-62)
            edges = edges[~((edges == 5).any(1) & (edges == 9).any(1))]
            edges[0] = (5, 9)
            X[5] = X[9]
            key = "m%d_zero" % m
        out[key + "/edges"] = edges
        out[key + "/X"] = X
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            cases = function_cases(p, dtype, np.random.default_rng(7))
            for name, (f, pars) in cases.items():
                mde = pymde.MDE(n, m, torch.tensor(edges), f, pymde.Centered())
                Xt = torch.tensor(X, dtype=dtype, requires_grad=True)
                v = mde.average_distortion(Xt)
                v.backward()
                out["%s/%s/%s/value" % (key, name, tag)] = v.detach().numpy()
                out["%s/%s/%s/grad" % (key, name, tag)] = Xt.grad.numpy()
                if m == 2 and tag == "f32" and not zero:
                    out["%s/%s/distances" % (key, name)] = mde.distances(Xt.detach()).numpy()
                    out["%s/%s/distortions" % (key, name)] = mde.distortions(Xt.detach()).numpy()
    np.savez_compressed(os.path.join(HERE, "evals.npz"), **out)
    print("evals.npz", len(out))


def gen_projections():
    out = {}
    rng = np.random.default_rng(3)
    std, cen = pymde.Standardized(), pymde.Centered()
    for (n, m) in ((2, 2), (10, 3), (100, 3), (1000, 2), (257, 5), (300, 40)):
        Z = rng.standard_normal((n, m)).astype(np.float32) + 0.3
        key = "n%d_m%d" % (n, m)
        out[key + "/Z"] = Z
        out[key + "/centered"] = cen.project_onto_constraint(torch.tensor(Z), inplace=False).numpy()
        Xs = std.project_onto_constraint(torch.tensor(Z).clone(), inplace=False)
        out[key + "/standardized"] = Xs.numpy()
        G = rng.standard_normal((n, m)).astype(np.float32)
        out[key + "/G"] = G
        out[key + "/tangent"] = std.project_onto_tangent_space(
            Xs, torch.tensor(G), inplace=False).numpy()
    np.savez_compressed(os.path.join(HERE, "projections.npz"), **out)
    print("projections.npz", len(out))


def knn_like_graph(n, k, rng):
    """Synthetic stand-in for a k-NN graph on a ring with a few chords (no datasets here)."""
    e = set()
    for i in range(n):
        for o in range(1, k + 1):
            j = (i + o) % n
            e.add((min(i, j), max(i, j)))
    for _ in range(n // 2):
        i, j = rng.integers(0, n, 2)
        if i != j:
            e.add((min(i, j), max(i, j)))
    return np.array(sorted(e), dtype=np.int64)


def gen_trajectories():
    out = {}
    pen, los = pymde.penalties, pymde.losses

    def run(key, n, m, edges, f, constraint, max_iter, X0=None, eps=1e-5, memory_size=10):
        mde = pymde.MDE(n, m, torch.tensor(edges), f, constraint)
        if X0 is None:
            torch.manual_seed(0)
            X0 = constraint.initialization(n, m)
        # float64 run of the same reference code (tensors stay float64 end to end): pins the
        # ALGORITHM (L-BFGS, Wolfe search, projections) free of fp32 summation-order noise
        f64 = f.double()
        mde64 = pymde.MDE(n, m, torch.tensor(edges), f64, constraint)
        X64 = mde64.embed(X=X0.double(), max_iter=max_iter, eps=eps, memory_size=memory_size)
        out[key + "/f64/X"] = X64.detach().numpy()
        out[key + "/f64/average_distortions"] = np.array(mde64.solve_stats.average_distortions)
        out[key + "/f64/residual_norms"] = np.array(mde64.solve_stats.residual_norms)
        out[key + "/f64/step_size_percents"] = np.array(mde64.solve_stats.step_size_percents)
        f.float()
        X = mde.embed(X=X0, max_iter=max_iter, eps=eps, memory_size=memory_size)
        st = mde.solve_stats
        out[key + "/edges"] = edges
        out[key + "/X0"] = X0.numpy()
        out[key + "/X"] = X.detach().numpy()
        out[key + "/average_distortions"] = np.array(st.average_distortions)
        out[key + "/residual_norms"] = np.array(st.residual_norms)
        out[key + "/step_size_percents"] = np.array(st.step_size_percents)
        out[key + "/final_value"] = mde.average_distortion(X.detach()).numpy()
        out[key + "/max_iter"] = np.array(max_iter)
        out[key + "/eps"] = np.array(eps)
        print(key, "iters", st.iterations, "value", float(out[key + "/final_value"]))

    rng = np.random.default_rng(5)
    # T1: quadratic + standardized (spectral problem; converges)
    n, m = 80, 2
    edges = knn_like_graph(n, 3, rng)
    w = np.ones(len(edges), np.float32)
    out["quad_std/par0"] = w
    run("quad_std", n, m, edges, pen.Quadratic(torch.tensor(w)), pymde.Standardized(), 60)
    # T2: push-and-pull Log1p/Log + centered (the preserve_neighbors default)
    n, m = 120, 2
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
    out["pp_cen/par0"] = w
    run("pp_cen", n, m, edges, pen.PushAndPull(torch.tensor(w), pen.Log1p, pen.Log),
        pymde.Centered(), 40)
    # T3: push-and-pull + standardized, m = 3
    out["pp_std/par0"] = w
    run("pp_std", n, 3, edges, pen.PushAndPull(torch.tensor(w), pen.Log1p, pen.Log),
        pymde.Standardized(), 40)
    # T4: C1-shaped: cycle graph, all pairs, hop distances, Absolute, centered (nonsmooth)
    n, m = 40, 2
    iu = np.triu_indices(n, 1)
    edges = np.stack(iu, 1).astype(np.int64)
    hop = np.minimum(edges[:, 1] - edges[:, 0], n - (edges[:, 1] - edges[:, 0])).astype(np.float32)
    out["cycle_abs/par0"] = hop
    run("cycle_abs", n, m, edges, los.Absolute(torch.tensor(hop)), pymde.Centered(), 40)
    # T5: C3-shaped: Huber loss + standardized on sampled pairs
    n, m = 100, 2
    edges = random_graph(n, 900, rng)
    delta = rng.integers(1, 6, len(edges)).astype(np.float32)
    delta = delta * (np.sqrt(2.0 * n * m / (n - 1)) / np.sqrt((delta ** 2).mean()))
    delta = delta.astype(np.float32)
    out["huber_std/par0"] = delta
    run("huber_std", n, m, edges, los.Huber(torch.tensor(delta), 0.5), pymde.Standardized(), 40)
    # T6: docs example (docs_src/source/mde/index.rst:193-286): 5 items, 4 edges
    edges = np.array([[0, 1], [0, 2], [0, 3], [3, 4]], dtype=np.int64)
    w = np.array([1.0, 2.0, 5.0, 6.0], np.float32)
    out["docs5/par0"] = w
    run("docs5", 5, 2, edges, pen.Quadratic(torch.tensor(w)), pymde.Standardized(), 100)
    np.savez_compressed(os.path.join(HERE, "trajectories.npz"), **out)
    print("trajectories.npz", len(out))


def gen_anchored():
    """Anchored constraint (pymde/constraints.py:114-164), the 'embedding new points' workflow: 12 anchors keep their
    values, the other rows are optimised.  (a) Quadratic penalties: converges (convex in the free rows);
    (b) PushAndPull(Log1p, Log): 40 iterations.  fp32 and fp64 runs of the unmodified reference."""
    out = {}
    pen = pymde.penalties
    rng = np.random.default_rng(21)
    n, m = 150, 2
    att = knn_like_graph(n, 4, rng)
    rep = random_graph(n, len(att), np.random.default_rng(22))
    anchors = np.sort(rng.choice(n, 12, replace=False)).astype(np.int64)
    values = rng.standard_normal((12, m)).astype(np.float32) * 2.0
    out["anchors"], out["values"] = anchors, values
    cases = {
        "quad": (att, np.ones(len(att), np.float32) * rng.uniform(0.5, 2.0, len(att)).astype(np.float32),
                 lambda w: pen.Quadratic(w), 200),
        "pp": (np.concatenate([att, rep]),
               np.concatenate([np.ones(len(att)), -np.ones(len(rep))]).astype(np.float32),
               lambda w: pen.PushAndPull(w, pen.Log1p, pen.Log), 40),
    }
    for key, (edges, w, mk, iters) in cases.items():
        out[key + "/edges"], out[key + "/par0"], out[key + "/max_iter"] = edges, w, np.array(iters)
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            cons = pymde.Anchored(torch.tensor(anchors), torch.tensor(values, dtype=dtype))
            if tag == "f32":
                torch.manual_seed(0)
                X0 = cons.initialization(n, m)
                out[key + "/X0"] = X0.numpy().copy()
            else:
                X0 = torch.tensor(out[key + "/X0"], dtype=dtype)
            mde = pymde.MDE(n, m, torch.tensor(edges), mk(torch.tensor(w, dtype=dtype)), cons)
            X = mde.embed(X=X0, max_iter=iters, eps=1e-6)
            st = mde.solve_stats
            out["%s/%s/X" % (key, tag)] = X.detach().numpy()
            out["%s/%s/average_distortions" % (key, tag)] = np.array(st.average_distortions)
            out["%s/%s/residual_norms" % (key, tag)] = np.array(st.residual_norms)
            out["%s/%s/final_value" % (key, tag)] = mde.average_distortion(X.detach()).numpy()
            print("anchored", key, tag, "iters", st.iterations, "final", float(out["%s/%s/final_value" % (key, tag)]))
    np.savez_compressed(os.path.join(HERE, "anchored.npz"), **out)
    print("anchored.npz", len(out))


def gen_nearzero():
    """Repulsive and attractive edges at tiny distances (VERDICT r01 weak item 3): the fast-math kernels switch to a
    series for 1 - exp(-d) below d = 0.0625 and mask d = 0; the reference (fp32 and fp64) is the arbiter.
    Points come in clusters of near-duplicates, so edge lengths span 1e-6 .. 1e-1 plus exact zeros."""
    out = {}
    pen = pymde.penalties
    for m in (2, 3):
        rng = np.random.default_rng(100 + m)
        n, p = 240, 640
        centers = rng.standard_normal((n // 8, m)).astype(np.float32)
        scale = 10.0 ** rng.uniform(-6, -1, n).astype(np.float32)
        X = (centers[np.arange(n) // 8] + scale[:, None] * rng.standard_normal((n, m)).astype(np.float32)).astype(np.float32)
        X[1] = X[0]            # exact duplicates: d = 0 on an attractive and on a repulsive edge
        X[9] = X[8]
        pairs = set()
        while len(pairs) < p - 2:
            c = int(rng.integers(0, n // 8))
            i, j = rng.integers(0, 8, 2) + 8 * c   # inside a cluster: tiny distance
            if rng.random() < 0.2:
                j = int(rng.integers(0, n))        # some ordinary lengths too
            if i != j and (min(i, j), max(i, j)) not in ((0, 1), (8, 9)):
                pairs.add((min(i, j), max(i, j)))
        edges = np.array(sorted(pairs) + [(0, 1), (8, 9)], dtype=np.int64)
        w = rng.choice([1.0, 2.0, -1.0], len(edges)).astype(np.float32)
        w[-2], w[-1] = 1.0, -1.0
        key = "m%d" % m
        out[key + "/edges"], out[key + "/X"], out[key + "/par0"] = edges, X, w
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            f = pen.PushAndPull(torch.tensor(w, dtype=dtype), pen.Log1p, pen.Log)
            mde = pymde.MDE(n, m, torch.tensor(edges), f, pymde.Centered())
            Xt = torch.tensor(X, dtype=dtype, requires_grad=True)
            d = mde.distances(Xt.detach())
            keep = d > 0   # the reference's VALUE is -inf on a zero-length repulsive edge; its gradient is defined
            v = mde.average_distortion(Xt)
            v.backward()
            out["%s/%s/grad" % (key, tag)] = Xt.grad.numpy()
            out["%s/%s/distances" % (key, tag)] = d.numpy()
            fk = f(d)
            out["%s/%s/value_nonzero_edges" % (key, tag)] = (fk[keep].sum() / len(edges)).numpy()
        print("nearzero", key, "min positive d", float(out[key + "/f64/distances"][out[key + "/f64/distances"] > 0].min()))
    np.savez_compressed(os.path.join(HERE, "nearzero.npz"), **out)
    print("nearzero.npz", len(out))


def gen_c2slice():
    """C2-scale slice (VERDICT r01 item 3a): the bench generator at n = 20 000 (444 024 edges, PushAndPull(Log1p, Log)).
    (i) Standardized, run by the reference to convergence (eps = 1e-5) with 1, 4 and 8 torch threads: the objective is
    non-convex and the fp32 scatter order depends on the thread count, so the reference itself converges to different
    stationary points -- the spread of its final values is part of the fixture; (ii) Centered, 300 iterations (not
    converged), 1 and 8 threads.  Edges are regenerated by bench.c2_edges (sha1 stored), only X0 / final X travel."""
    import hashlib
    import bench
    out = {}
    n, m = 20000, 2
    edges, w = bench.c2_edges(0, n=n, k=15)
    X0 = bench.initial_iterate(0, n=n)
    out["edges_sha1"] = np.frombuffer(hashlib.sha1(edges.tobytes() + w.tobytes()).digest(), dtype=np.uint8)
    out["n_edges"] = np.array(len(edges))
    pen = pymde.penalties
    cons = pymde.Standardized()
    Xs = cons.project_onto_constraint(torch.tensor(X0).clone())
    out["std/X0"] = Xs.numpy().copy()
    for th in (8, 4, 1):
        torch.set_num_threads(th)
        mde = pymde.MDE(n, m, torch.tensor(edges), pen.PushAndPull(torch.tensor(w), pen.Log1p, pen.Log), cons)
        X = mde.embed(X=Xs.clone(), max_iter=1500, eps=1e-5)
        st = mde.solve_stats
        out["std/t%d/average_distortions" % th] = np.array(st.average_distortions)
        out["std/t%d/residual_norms" % th] = np.array(st.residual_norms)
        out["std/t%d/final_value" % th] = mde.average_distortion(X.detach()).numpy()
        if th == 8:
            out["std/t8/X"] = X.detach().numpy().copy()
        print("c2slice std threads", th, "iters", st.iterations, "final", float(out["std/t%d/final_value" % th]))
    out["cen/X0"] = X0
    for th in (8, 1):
        torch.set_num_threads(th)
        mde = pymde.MDE(n, m, torch.tensor(edges), pen.PushAndPull(torch.tensor(w), pen.Log1p, pen.Log), pymde.Centered())
        mde.embed(X=torch.tensor(X0), max_iter=300, eps=1e-5)
        st = mde.solve_stats
        out["cen/t%d/average_distortions" % th] = np.array(st.average_distortions)
        out["cen/t%d/residual_norms" % th] = np.array(st.residual_norms)
        print("c2slice cen threads", th, "iters", st.iterations, "last", st.average_distortions[-1])
    torch.set_num_threads(1)
    np.savez_compressed(os.path.join(HERE, "c2slice.npz"), **out)
    print("c2slice.npz", len(out))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "c2slice":
        gen_c2slice()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "anchored":
        gen_anchored()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "nearzero":
        gen_nearzero()
        sys.exit(0)
    gen_functions()
    gen_evals()
    gen_projections()
    gen_trajectories()
    gen_anchored()
    gen_nearzero()
    gen_c2slice()
