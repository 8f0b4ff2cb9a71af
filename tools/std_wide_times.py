#!/usr/bin/env python
"""Standardized embeddings wider than 256 columns: the device solver against the host-stepped path it replaces.

C2-shaped problems (bench.py's edges, n = 70 000, PushAndPull(Log1p, Log)) with Standardized() at each width.  For
each width:

  device   ms per embed() iteration on the device-resident solver (mde.embed, eps = 0), CUDA events around the call
  host     ms per iteration of generic_solver.lbfgs_generic with a Constraint subclass whose projections are the torch
           branches the device path replaced: the retraction through an fp64 Gram and torch.linalg.eigh (cuSOLVER),
           the tangent projection as two fp32 GEMMs
  the two alternate in one call, `--repeats` windows each after one warm-up; best and spread ((max - min) / best)

then, from the library's own entries on a standardized X near the solver's trial points:

  retraction / tangent   ms per mde_project_standardized / mde_tangent_standardized call (CUDA events, 20 calls)
  kernels                per-launch times from torch.profiler: gram_wide_kernel at 2 n m^2 flops per launch,
                         rowgemm_kernel at 2 n m^2 over the launches of one call (one per chunk of rows; with the
                         retraction's copy_kernel reported apart), ns_init_kernel as a time, ns_dmma_kernel at 2 m^3 per product (the residual launch computes one, the
                         update launch two), timed on a retraction of a cond(X_c) = 1e3 input, where the chain runs
                         about 23 of its 24 iterations; launches the convergence gate switched off (shorter than half
                         the longest of their kind) are left out.  Rates against the data sheet's 67 TFLOP/s FP32
                         (FFMA) and 67 TFLOP/s FP64 tensor core.

The card's name, power limit and SM clock cap are read in the same call.

    python tools/std_wide_times.py [--widths 260,300,512,1024] [--iters K] [--host-iters K] [--repeats R]
                                   [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

PEAK_FP32 = 67e12
PEAK_FP64_TC = 67e12


def torch_standardized(torch, pm):
    """Standardized with the torch projections the device entries replace for 256 < m <= 1024."""
    class TorchStandardized(pm.constraints.Constraint):
        def name(self):
            return "standardized (torch eigh + GEMM)"

        def initialization(self, n_items, embedding_dim, device=None):
            return self.project_onto_constraint(torch.randn((int(n_items), int(embedding_dim)), device=device))

        def project_onto_constraint(self, Z, inplace=True):
            out = Z if inplace else Z.detach().clone()
            n = out.shape[0]
            with torch.no_grad():
                D = out.double()
                D = D - D.mean(dim=0)
                lam, Q = torch.linalg.eigh(D.T @ D)
                if not bool(lam[0] > 1e-12 * lam[-1]):
                    raise pm.util.SolverError("Gram matrix is not positive definite")
                W = (Q * lam.rsqrt()) @ Q.T * (float(n) ** 0.5)
                out.copy_((D @ W).float())
            return out

        def project_onto_tangent_space(self, X, Z, inplace=True):
            out = Z if inplace else Z.detach().clone()
            with torch.no_grad():
                out.sub_((1.0 / out.shape[0]) * (X @ (out.T @ X)))
            return out

    return TorchStandardized()


def events_ms(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_rates(torch, lib, X, ws, stream, n, m):
    """Per-launch times of the wide kernels over one retraction and one tangent projection (profiler)."""
    from torch.autograd import DeviceType
    Z = torch.randn_like(X)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        Y = X.clone()
        lib.mde_project_standardized(Y.data_ptr(), n, m, ws.data_ptr(), stream)
        lib.mde_tangent_standardized(Y.data_ptr(), Z.data_ptr(), n, m, ws.data_ptr(), stream)
        torch.cuda.synchronize()
    launches = {}
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        for key in ("gram_wide_kernel", "rowgemm_kernel", "ns_dmma_kernel<true>", "ns_dmma_kernel<false>",
                    "ns_init_kernel", "copy_kernel"):
            if key in e.name:
                launches.setdefault(key, []).append(e.time_range.elapsed_us() * 1e-6)
    flops = {"gram_wide_kernel": 2.0 * n * m * m, "rowgemm_kernel": 2.0 * n * m * m,
             "ns_dmma_kernel<true>": 2.0 * m ** 3, "ns_dmma_kernel<false>": 4.0 * m ** 3}
    out = {}
    for key, ts in launches.items():
        ts = np.array(ts)
        if key not in flops:  # no arithmetic to rate: time only
            out[key] = {"launches": int(len(ts)), "us_total": round(float(ts.sum()) * 1e6, 2)}
            continue
        run = ts[ts >= 0.5 * ts.max()] if key.startswith("ns_") else ts
        calls = len(run)
        if key == "rowgemm_kernel":  # one launch per chunk of rows, in each of the two calls profiled
            calls = 2
        rate = flops[key] * calls / run.sum()
        out[key] = {"launches": int(len(ts)), "timed": int(len(run)), "us_per_launch": round(float(run.mean()) * 1e6, 2),
                    "tflops": round(rate / 1e12, 2), "share_of_67tf": round(rate / (PEAK_FP64_TC if key.startswith("ns_")
                                                                                   else PEAK_FP32), 3)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--widths", default="260,300,512,1024")
    ap.add_argument("--iters", type=int, default=30, help="iterations per timed device embed()")
    ap.add_argument("--host-iters", type=int, default=10, help="iterations per timed host-stepped solve")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import bench
    import pymde_b200 as pm
    from pymde_b200 import _lib, util
    from pymde_b200.generic_solver import lbfgs_generic
    from tests.test_gpu_projections import _input

    if not torch.cuda.is_available():
        raise SystemExit("std_wide_times.py measures on a CUDA device; none found")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib = _lib.load()
    gpu = bench.gpu_identity(dev)
    print("GPU: %s, power limit %s W, SM clock cap %s MHz" % (gpu["name"], gpu["power_limit_w"], gpu["sm_max_mhz"]))
    edges, w = bench.c2_edges(0)
    n = bench.N_ITEMS
    E = torch.tensor(edges, device=dev)
    wt = torch.tensor(w, device=dev)
    host_cons = torch_standardized(torch, pm)
    rows = []
    for m in [int(v) for v in args.widths.split(",")]:
        f = pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log)
        mde = pm.MDE(n, m, E, f, pm.Standardized(), device=dev)
        assert mde._fused_ok(mde.constraint, 10), m
        torch.manual_seed(m)
        X0 = pm.Standardized().initialization(n, m, dev)

        def device_arm():
            X = X0.clone()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            mde.embed(X=X, max_iter=args.iters, eps=0.0)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / mde.solve_stats.iterations

        def host_arm():
            X = X0.clone()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _, st = lbfgs_generic(X, mde.average_distortion, host_cons, 0.0, args.host_iters, 10, True, True, False,
                                  args.host_iters, None, pm.problem.LOGGER)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / st.iterations

        device_arm()
        host_arm()
        dev_ms, host_ms = [], []
        for _ in range(args.repeats):
            dev_ms.append(device_arm())
            host_ms.append(host_arm())

        # the entries on a standardized X (the solver's trial points are this close)
        Xs = util.proj_standardized(X0.clone(), demean=True)
        ws = torch.empty(lib.mde_project_ws_bytes(n, m), dtype=torch.uint8, device=dev)
        stream = util.stream_ptr(dev)
        Y = Xs.clone()
        Z = torch.randn_like(Xs)
        retr = events_ms(torch, lambda: lib.mde_project_standardized(Y.data_ptr(), n, m, ws.data_ptr(), stream), 20)
        tang = events_ms(torch, lambda: lib.mde_tangent_standardized(Xs.data_ptr(), Z.data_ptr(), n, m, ws.data_ptr(),
                                                                     stream), 20)
        kr = kernel_rates(torch, lib, _input(n, m, "cond1e3", m), ws, stream, n, m)
        r = {"m": m, "n": n, "p": int(len(edges)),
             "device_ms_per_iter": {"best": round(min(dev_ms), 3), "spread": round((max(dev_ms) - min(dev_ms)) / min(dev_ms), 3),
                                    "windows": [round(v, 3) for v in dev_ms]},
             "host_ms_per_iter": {"best": round(min(host_ms), 3), "spread": round((max(host_ms) - min(host_ms)) / min(host_ms), 3),
                                  "windows": [round(v, 3) for v in host_ms]},
             "speedup_best": round(min(host_ms) / min(dev_ms), 2),
             "retraction_ms": round(retr, 4), "tangent_ms": round(tang, 4), "kernels": kr}
        rows.append(r)
        print(json.dumps(r), flush=True)
        del mde
        torch.cuda.empty_cache()
    res = {"gpu": gpu, "iters": args.iters, "host_iters": args.host_iters, "repeats": args.repeats, "rows": rows}
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
