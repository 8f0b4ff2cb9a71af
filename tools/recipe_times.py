"""Stage times of the recipes on a data matrix, with the graph assembled on the device or in a host scipy Graph, and
the neighbour-graph builder against the torch sort + unique_consecutive form it replaced (DESIGN section 11.5).

    python tools/recipe_times.py [--out FILE.json] [--quick] [--skip-10m]

Stages: search (neighbour search or pair distances), graph (assembly into the edge list, device copies included),
spectral (quadratic initialisation), negatives (sample_edges), mde (MDE construction), embed (embed(max_iter=300)).
The two arms alternate, and every timed pair is checked bit for bit: edges, weights / deviations and X_init.  Each
stage is timed by a host clock between device synchronisations.  The card's name and power limit are read in the
same run and written with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pymde_b200 as pm  # noqa: E402
from pymde_b200 import preprocess, problem, quadratic  # noqa: E402
from pymde_b200.preprocess import data_matrix as dm, graph as G  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:  # (the measurement itself needs the device, not nvidia-smi)
        out = "unknown (%s)" % exc
    return out


def mixture(n, d, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centers = torch.randn(10, d, device="cuda", generator=g) * 3
    lab = torch.randint(0, 10, (n,), device="cuda", generator=g)
    return (centers[lab] + torch.randn(n, d, device="cuda", generator=g)).cpu().numpy()


class Stages:
    """Accumulated wall time of wrapped functions (device synchronised on entry and exit); nested calls of a wrapped
    function are charged to the outer one only."""

    def __init__(self):
        self.t, self._depth = {}, {}

    def wrap(self, owner, name, label):
        fn = getattr(owner, name)
        is_static = isinstance(owner, type) and isinstance(owner.__dict__.get(name), staticmethod)

        def timed(*a, **kw):
            if self._depth.get(label):
                return fn(*a, **kw)
            self._depth[label] = 1
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                return fn(*a, **kw)
            finally:
                torch.cuda.synchronize()
                self.t[label] = self.t.get(label, 0.0) + time.perf_counter() - t0
                self._depth[label] = 0
        setattr(owner, name, staticmethod(timed) if is_static else timed)
        return lambda: setattr(owner, name, staticmethod(fn) if is_static else fn)


def run_recipe(make, arm, seed):
    st = Stages()
    undo = []
    if arm == "host":
        knn0, dist0 = dm.k_nearest_neighbors_device, dm.distances_device
        dm.k_nearest_neighbors_device = lambda data, k, max_distance=None, device=None: dm.k_nearest_neighbors(
            data, k, max_distance=max_distance, device=device)
        dm.distances_device = lambda data, retain_fraction=1.0, device=None: dm.distances(
            data, retain_fraction=retain_fraction, device=device)
        undo.append(lambda: setattr(dm, "k_nearest_neighbors_device", knn0))
        undo.append(lambda: setattr(dm, "distances_device", dist0))
    undo += [st.wrap(dm, "_search", "search"), st.wrap(dm, "_pair_distances", "search"),
             st.wrap(dm, "k_nearest_neighbors_device", "build"), st.wrap(dm, "distances_device", "build"),
             st.wrap(G.Graph, "_materialise", "materialise"), st.wrap(quadratic, "spectral", "spectral"),
             st.wrap(preprocess, "sample_edges", "negatives"), st.wrap(problem.MDE, "__init__", "mde")]
    try:
        pm.seed(seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mde = make()
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        for u in reversed(undo):
            u()
    t = st.t
    stages = {"search": t.get("search", 0.0), "graph": t.get("build", 0.0) - t.get("search", 0.0) +
              t.get("materialise", 0.0), "spectral": t.get("spectral", 0.0), "negatives": t.get("negatives", 0.0),
              "mde": t.get("mde", 0.0), "recipe": total}
    f = mde.distortion_function
    key = (mde.edges.clone(), (f.weights if hasattr(f, "weights") else f.deviations).clone(),
           getattr(mde, "_X_init", None))
    return mde, stages, key


def same(a, b):
    return all((x is None and y is None) or (x is not None and y is not None and torch.equal(x, y))
               for x, y in zip(a, b))


def time_embed(mde):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mde.embed(max_iter=300)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def shape(name, make, reps, arms=("host", "device")):
    rows = {a: [] for a in arms}
    parity = True
    for r in range(reps):
        keys = {}
        for arm in (arms if r % 2 == 0 else tuple(reversed(arms))):
            mde, stages, keys[arm] = run_recipe(make, arm, seed=r)
            stages["embed"] = time_embed(mde)
            rows[arm].append(stages)
            del mde
            torch.cuda.empty_cache()
        if len(arms) == 2:
            parity &= same(keys["host"], keys["device"])
        print(name, r, {a: {k: round(v, 4) for k, v in rows[a][-1].items()} for a in arms}, flush=True)
    med = {a: {k: float(np.median([s[k] for s in rows[a]])) for k in rows[a][0]} for a in arms}
    return {"reps": reps, "median_s": med, "bit_parity": parity if len(arms) == 2 else None}


def torch_form(idx, n):
    """k_nearest_neighbors_device's assembly before the builder: sort the canonical 64-bit keys, count the runs."""
    k = idx.shape[1]
    dst = idx.reshape(-1).long()
    src = torch.arange(n, device=idx.device).repeat_interleave(k)
    found = dst >= 0
    src, dst = src[found], dst[found]
    key = torch.minimum(src, dst) * n + torch.maximum(src, dst)
    key, counts = torch.unique_consecutive(torch.sort(key)[0], return_counts=True)
    return torch.stack([key // n, key % n], 1), counts.float()


def builder_ab(n, k, hub=False, reps=3):
    g = torch.Generator(device="cuda").manual_seed(n + k)
    idx = ((torch.arange(n, device="cuda")[:, None] + torch.randint(1, n, (n, k), device="cuda", generator=g)) % n)
    idx = idx.int()
    if hub:
        idx[:, 3] = 7
        idx[7, 3] = 8
    out = {}
    results = {}
    arms = (("builder", lambda: G.knn_edge_list(idx, n)), ("torch", lambda: torch_form(idx, n)))
    for r in range(reps):
        for name, fn in (arms if r % 2 == 0 else arms[::-1]):
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            res = fn()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            peak = torch.cuda.max_memory_allocated() - base
            res = (res.edges, res.weights) if name == "builder" else res
            if r == 0:
                results[name] = res
            o = out.setdefault(name, {"s": [], "peak_gb": 0.0})
            o["s"].append(dt)
            o["peak_gb"] = max(o["peak_gb"], peak / 1e9)
            del res
    parity = torch.equal(results["builder"][0], results["torch"][0]) and torch.equal(results["builder"][1],
                                                                                    results["torch"][1])
    p = int(results["builder"][0].shape[0])
    del results
    summary = {name: {"median_s": float(np.median(o["s"][1:] or o["s"])), "peak_gb": o["peak_gb"]}
               for name, o in out.items()}
    print("builder A/B n=%d k=%d hub=%s p=%d" % (n, k, hub, p), summary, "parity", parity, flush=True)
    return {"n": n, "k": k, "hub": hub, "pairs": p, "bit_parity": parity, **summary}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    ap.add_argument("--quick", action="store_true", help="small shapes only (a rehearsal)")
    ap.add_argument("--skip-10m", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "recipe_times.py measures on the GPU"
    res = {"card": card(), "torch": torch.__version__}
    print(res, flush=True)
    # warm-up, untimed: module loads and library set-up of every stage, in both arms
    W = mixture(3000, 784)
    for arm in ("host", "device"):
        for make in (lambda: pm.preserve_neighbors(W), lambda: pm.preserve_distances(W)):
            time_embed(run_recipe(make, arm, 0)[0])
    del W
    big = 20000 if args.quick else 10 ** 6
    # builder A/B
    res["builder_ab"] = []
    for n in ((big,) if args.quick else (10 ** 6, 10 ** 7)):
        for k in (15, 64):
            res["builder_ab"].append(builder_ab(n, k))
    res["builder_ab"].append(builder_ab(big, 15, hub=True))
    # recipes
    n_a = 5000 if args.quick else 70000
    X = mixture(n_a, 784)
    res["a_preserve_neighbors_70k_784"] = shape("a", lambda: pm.preserve_neighbors(X), 1 if args.quick else 3)
    res["b_preserve_distances_70k_784"] = shape("b", lambda: pm.preserve_distances(X), 1 if args.quick else 2)
    del X
    os.environ["PYMDE_B200_KNN"] = "approx"
    Y = mixture(big, 50, seed=1)
    res["c_preserve_neighbors_1m_50_approx"] = shape("c", lambda: pm.preserve_neighbors(Y), 1 if args.quick else 2)
    del Y
    if not args.skip_10m and not args.quick:
        Z = mixture(10 ** 7, 50, seed=2)
        res["d_preserve_neighbors_10m_50_approx"] = shape("d", lambda: pm.preserve_neighbors(Z), 1, arms=("device",))
        del Z
    os.environ.pop("PYMDE_B200_KNN")
    res["card_after"] = card()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
