#!/usr/bin/env python
"""A/B of the two evaluations at m >= 5: the default wide push kernel (float reds) and the deterministic wide owner
kernel (MDE_B200_DETERMINISTIC=1: owner-complete rows, no atomics).

    python tools/wide_owner_ab.py [--shapes c4slice,c4,c2m8,c2m16,c2m32,hub] [--rounds 3] [--quick] [--out FILE]

Both layouts are built in one process (the switch is read when a layout is created) and the arms alternate, `--rounds`
times.  Per shape and arm:
  warm_us     mde_distortion (fused value + gradient) alone, X and layout L2-resident: 50 launches between two events
  cold_us     the same with a 512 MB write before each launch, mean of 10 launches timed one by one
  step_ms     embed() with the device solver: 20 iterations after a 5-iteration warm-up, host clock around a synchronise,
              per iteration
and once per shape the parity of the arms at X0: value (relative) and gradient (max abs difference over max |g|),
checked against 1e-5 and 3e-5.  The card's name and power limit are read in the same process and printed first.

Shapes: c4slice (n = 2e5, m = 128, 8 neighbours + 8 negatives per node, the C4 slice of tests/test_gpu_configs.py),
c4 (n = 1e6, m = 128, 15 + 15 per node, about 3e7 edges), c2mM (bench.py's C2 graph, n = 70 000, at m = M), hub (the C4
slice plus one node of degree 1.2e5).  `--quick` rehearses at n = 3 000.  There is no CPU path."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc


def make_shape(torch, name, quick):
    """(n, m, edges (p, 2) int64 on the device, weights (p,) on the device)."""
    dev = "cuda"
    gen = torch.Generator(device=dev)
    gen.manual_seed(1)

    def knn_like(n, k, span):
        i = torch.arange(n, device=dev).repeat_interleave(k)
        j = (i + torch.randint(1, span, (i.numel(),), device=dev, generator=gen)) % n
        rep = torch.randint(0, n, (i.numel(), 2), device=dev, generator=gen)
        rep = rep[rep[:, 0] != rep[:, 1]]
        e = torch.cat([torch.stack([i, j], 1), rep])
        w = torch.cat([torch.ones(i.numel(), device=dev), -torch.ones(rep.shape[0], device=dev)])
        return e, w

    if name.startswith("c2m"):
        import bench
        m = int(name[3:])
        n = 3000 if quick else bench.N_ITEMS
        edges, w = bench.c2_edges(0, n=n) if quick else bench.c2_edges(0)
        return n, m, torch.tensor(edges, device=dev), torch.tensor(w, device=dev)
    if name == "c4":
        n = 3000 if quick else 1_000_000
        e, w = knn_like(n, 15, min(1000, n - 1))
        return n, 128, e, w
    n = 3000 if quick else 200_000
    e, w = knn_like(n, 8, min(1000, n - 1))
    if name == "hub":
        deg = 1000 if quick else 120_000
        hub = torch.stack([torch.zeros(deg, dtype=torch.int64, device=dev),
                           torch.randint(1, n, (deg,), device=dev, generator=gen)], 1)
        e = torch.cat([e, hub])
        w = torch.cat([w, torch.ones(deg, device=dev)])
    return n, 128, e, w


def build(pm, torch, n, m, e, w, det):
    if det:
        os.environ["MDE_B200_DETERMINISTIC"] = "1"
    else:
        os.environ.pop("MDE_B200_DETERMINISTIC", None)
    try:
        f = pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log)
        mde = pm.MDE(n, m, e, f, pm.Centered(), device="cuda")
        lay = mde._layout()  # the switch is read here
    finally:
        os.environ.pop("MDE_B200_DETERMINISTIC", None)
    from pymde_b200 import _lib
    assert int(_lib.load().mde_edges_deterministic(lay.handle)) == int(det)
    return mde, lay


def kernel_times(torch, lay, X, flush):
    from pymde_b200 import _lib, util
    lib = _lib.load()
    grad = torch.zeros_like(X)
    st = util.stream_ptr(X.device)

    def launch():
        _lib.check(lib.mde_distortion(lay.handle, X.data_ptr(), X.shape[1], grad.data_ptr(), None, st))

    for _ in range(3):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(50):
        launch()
    b.record()
    torch.cuda.synchronize()
    warm = a.elapsed_time(b) * 1e3 / 50
    cold = []
    for _ in range(10):
        flush.fill_(1.0)
        a.record()
        launch()
        b.record()
        torch.cuda.synchronize()
        cold.append(a.elapsed_time(b) * 1e3)
    return warm, float(np.mean(cold))


def step_time(torch, mde, X0):
    mde.embed(X=X0.clone(), max_iter=5, eps=0.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mde.embed(X=X0.clone(), max_iter=20, eps=0.0)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / max(1, mde.solve_stats.iterations)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c4slice,c4,c2m8,c2m16,c2m32,hub")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--no-step", action="store_true", help="skip the embed() step times")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("wide_owner_ab.py measures on a CUDA device; none is available")
    import pymde_b200 as pm
    info = gpu_info()
    print("gpu: %s" % info, flush=True)
    flush = torch.empty(128 * 1024 * 1024, device="cuda")  # 512 MB
    results = {"gpu": info, "shapes": {}}
    for name in args.shapes.split(","):
        n, m, e, w = make_shape(torch, name, args.quick)
        arms = {"wide": build(pm, torch, n, m, e, w, False), "owner": build(pm, torch, n, m, e, w, True)}
        gen = torch.Generator(device="cuda")
        gen.manual_seed(2)
        X0 = torch.randn(n, m, device="cuda", generator=gen)
        X0 -= X0.mean(0)
        vals = {k: lay.value_and_grad(X0) for k, (_, lay) in arms.items()}
        (vw, gw), (vo, go) = vals["wide"], vals["owner"]
        rel_v = abs(vo.item() - vw.item()) / abs(vw.item())
        rel_g = float((go - gw).abs().max()) / float(gw.abs().max())
        rec = {"n": n, "m": m, "p": int(e.shape[0]), "value_rel_diff": rel_v, "grad_diff_over_max": rel_g,
               "parity_ok": bool(rel_v <= 1e-5 and rel_g <= 3e-5), "rounds": []}
        print("%s: n=%d m=%d p=%d  value rel diff %.2e  grad diff/max %.2e  parity %s" % (
            name, n, m, rec["p"], rel_v, rel_g, "ok" if rec["parity_ok"] else "FAILED"), flush=True)
        del vals, gw, go
        for r in range(args.rounds):
            row = {}
            for arm in (("wide", "owner") if r % 2 == 0 else ("owner", "wide")):
                mde, lay = arms[arm]
                warm, cold = kernel_times(torch, lay, X0, flush)
                step = None if args.no_step else step_time(torch, mde, X0)
                row[arm] = {"warm_us": warm, "cold_us": cold, "step_ms": step}
            rec["rounds"].append(row)
            print("  round %d  " % r + "  ".join(
                "%s: warm %.1f us, cold %.1f us, step %s ms" % (
                    a, row[a]["warm_us"], row[a]["cold_us"], "-" if row[a]["step_ms"] is None else "%.3f" % row[a]["step_ms"])
                for a in ("wide", "owner")), flush=True)
        results["shapes"][name] = rec
        del arms
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
