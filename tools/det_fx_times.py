"""Cost of deterministic mode at m <= 4 (MDE_B200_DETERMINISTIC=1): the fused evaluation and a 200-iteration solve
with the fixed-point accumulator, against an older build of the library (`--base`) and against the default mode.

  python tools/det_fx_times.py --base path/to/older/libmde_b200.so [--rounds 3] [--out FILE]

Shapes: the C2 graph shape (n = 70 000, 1.55e6 random edges) and n = 450 000 with 1e7 random edges, m = 2,
PushAndPull(Log1p, Log) with weights +-1, Centered.  Evaluation: `mde_distortion` (value and gradient), CUDA events
around each call, median of 50 after 5 warm-up calls.  Solve: `embed(max_iter=200, eps=1e-12)` from a fixed X0,
wall clock around a call that ends in a device synchronise, after one warm-up solve.  Every arm runs in a process of
its own (the library is loaded once per process); arms alternate for --rounds rounds.  The deterministic solve's final
average distortion is printed per arm, so the builds can be compared.  Prints the GPU's name, power limit and maximum
SM clock, then one JSON object."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
SHAPES = {"c2": (70_000, 1_550_000), "1e7": (450_000, 10_000_000)}


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True).stdout.strip()


def arm(lib_path, shapes, quick):
    """one arm in this process: {shape: {mode: {eval_ms, solve_s, distortion}}}"""
    sys.path.insert(0, ROOT)
    import torch
    from pymde_b200 import _lib, util
    if lib_path:
        _lib.LIB_PATH = os.path.abspath(lib_path)
    import pymde_b200 as pm
    lib = _lib.load()
    out = {}
    for shape in shapes:
        n, p = SHAPES[shape]
        if quick:
            n, p = 3_000, 60_000
        rng = np.random.default_rng(1)
        i = rng.integers(0, n, p)
        edges = torch.tensor(np.stack([i, (i + rng.integers(1, n, p)) % n], 1), device="cuda")
        w = torch.tensor(np.where(rng.random(p) < 0.5, 1.0, -1.0).astype(np.float32), device="cuda")
        f = pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log)
        X0 = torch.randn(n, 2, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        res = {}
        for mode in ("default", "det"):
            if mode == "det":
                os.environ["MDE_B200_DETERMINISTIC"] = "1"
            else:
                os.environ.pop("MDE_B200_DETERMINISTIC", None)
            mde = pm.MDE(n, 2, edges, f, pm.Centered(), device="cuda")
            lay = mde._layout()
            assert int(lib.mde_edges_deterministic(lay.handle)) == (mode == "det")
            grad = torch.zeros_like(X0)
            st = util.stream_ptr(X0.device)

            def call():
                grad.zero_()
                _lib.check(lib.mde_distortion(lay.handle, X0.data_ptr(), 2, grad.data_ptr(), lay.loss.data_ptr(), st))

            for _ in range(5):
                call()
            ts = []
            for _ in range(50):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call()
                b.record()
                b.synchronize()
                ts.append(a.elapsed_time(b))
            iters = 5 if quick else 200
            mde.embed(X=X0.clone(), max_iter=iters, eps=1e-12)  # warm-up of the solver at this shape
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mde.embed(X=X0.clone(), max_iter=iters, eps=1e-12)
            torch.cuda.synchronize()
            res[mode] = {"eval_ms": float(np.median(ts)), "solve_s": time.perf_counter() - t0,
                         "iterations": int(mde.solve_stats.iterations),
                         "distortion": float(mde.solve_stats.average_distortions[-1])}
            del mde, lay
            torch.cuda.empty_cache()
        os.environ.pop("MDE_B200_DETERMINISTIC", None)
        out[shape] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default=None, help="an older build of libmde_b200.so")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="c2,1e7")
    ap.add_argument("--quick", action="store_true", help="rehearse at n = 3 000")
    ap.add_argument("--out", default=None)
    ap.add_argument("--arm", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    shapes = a.shapes.split(",")
    if a.arm is not None:
        print("ARM " + json.dumps(arm(a.arm or None, shapes, a.quick)))
        return
    arms = ([("base", a.base)] if a.base else []) + [("tree", "")]
    runs = {name: [] for name, _ in arms}
    for _ in range(a.rounds):
        for name, path in arms:
            cmd = [sys.executable, os.path.abspath(__file__), "--arm", path, "--shapes", a.shapes]
            if a.quick:
                cmd.append("--quick")
            r = subprocess.run(cmd, capture_output=True, text=True, check=True)
            line = [s for s in r.stdout.splitlines() if s.startswith("ARM ")][-1]
            runs[name].append(json.loads(line[4:]))
    summary = {}
    for name, rs in runs.items():
        for shape in shapes:
            for mode in ("default", "det"):
                e = [r[shape][mode]["eval_ms"] for r in rs]
                s = [r[shape][mode]["solve_s"] for r in rs]
                summary["%s/%s/%s" % (name, shape, mode)] = {
                    "eval_ms": [min(e), max(e)], "solve_s": [min(s), max(s)],
                    "iterations": rs[0][shape][mode]["iterations"],
                    "distortion": [r[shape][mode]["distortion"] for r in rs]}
    print(_gpu())
    print(json.dumps(summary, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"gpu": _gpu(), "summary": summary, "runs": runs}, fh, indent=1)


if __name__ == "__main__":
    main()
