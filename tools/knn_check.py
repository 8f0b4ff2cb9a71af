"""mde_knn (wgmma cross terms + running top-32 + exact re-rank) against an fp64 brute force, and timed against the
library-GEMM + torch.topk path it replaces.  Usage: python tools/knn_check.py [small|full]"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pymde_b200.preprocess import data_matrix as dm

dev = torch.device("cuda", 0)


def brute64(X, rows, k):
    """k smallest fp64 squared distances (and indices) of the given rows."""
    Xd = X.double()
    Q = Xd[rows]
    d2 = (Q * Q).sum(1)[:, None] + (Xd * Xd).sum(1)[None, :] - 2.0 * Q @ Xd.T
    d2[torch.arange(len(rows), device=X.device), rows] = float("inf")
    val, idx = torch.topk(d2, k, dim=1, largest=False)
    return val, idx


def gemm_path(X, k, rows=8192):
    sq = (X * X).sum(1)
    out = []
    for s0 in range(0, X.shape[0], rows):
        Q = X[s0:s0 + rows]
        d2 = (sq[s0:s0 + rows, None] + sq[None, :] - 2.0 * (Q @ X.T)).clamp_(min=0)
        d2[torch.arange(Q.shape[0], device=X.device), torch.arange(s0, s0 + Q.shape[0], device=X.device)] = float("inf")
        out.append(torch.topk(d2, k, dim=1, largest=False)[1])
    return torch.cat(out)


def check(n, d, k, seed, clustered, time_it=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    if clustered:  # MNIST-like: non-negative, many exact zeros, cluster structure
        centers = torch.rand((10, d), generator=g, device=dev)
        lab = torch.randint(0, 10, (n,), generator=g, device=dev)
        X = (centers[lab] + 0.35 * torch.randn((n, d), generator=g, device=dev)).clamp_(0, 1)
        X = torch.where(X < 0.3, torch.zeros_like(X), X).contiguous()
    else:
        X = torch.randn((n, d), generator=g, device=dev)
    idx, d2 = dm.knn_device(X, k)
    torch.cuda.synchronize()
    rows = torch.arange(n, device=dev) if n <= 8192 else torch.randperm(n, generator=g, device=dev)[:4096]
    val, ref = brute64(X, rows, k)
    got = idx[rows].long()
    # exact fp64 distances of what we returned, in the returned order
    gd = ((X[rows].double()[:, None, :] - X[got].double()) ** 2).sum(-1)
    ok_sorted = bool((gd[:, 1:] >= gd[:, :-1] - 1e-6 * gd[:, 1:].abs() - 1e-9).all())
    rel = ((gd - val).abs() / val.clamp_min(1e-12)).max().item()
    same = (torch.sort(got, 1)[0] == torch.sort(ref, 1)[0]).all(1).float().mean().item()
    d2rel = ((d2[rows].double() - gd).abs() / gd.clamp_min(1e-12)).max().item()
    rec = {"n": n, "d": d, "k": k, "clustered": clustered, "rows_checked": int(len(rows)),
           "kth_distance_max_rel_err_vs_fp64": rel, "rows_with_identical_sets": same, "ascending": ok_sorted,
           "returned_d2_max_rel_err": d2rel, "self_in_list": bool((got == rows[:, None]).any())}
    if time_it:
        for name, fn in (("kernel_ms", lambda: dm.knn_device(X, k)), ("gemm_topk_ms", lambda: gemm_path(X, k))):
            fn(); torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
            rec[name] = min(ts)
        flops = 3 * 2.0 * n * n * ((d + 63) // 64 * 64)
        rec["tensor_tflops_at_kernel_ms"] = flops / (rec["kernel_ms"] * 1e-3) / 1e12
    print(json.dumps(rec), flush=True)
    return rec


mode = sys.argv[1] if len(sys.argv) > 1 else "small"
check(1000, 64, 5, 0, False)
check(3000, 100, 15, 1, False)
check(5000, 784, 15, 2, True)
if mode == "full":
    check(70000, 784, 15, 3, True, time_it=True)
