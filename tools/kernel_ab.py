#!/usr/bin/env python
"""A/B of the fused distortion kernel on one GPU: sorted-SoA layout (quad kernel, r01) against the tile-record
layouts (tile / pull / ELL-pull kernels, r02), cold L2 (512 MB flush before every launch), CUDA events, plus a parity check of the
two results against each other (loss to 1e-6 relative, gradient to 2e-5 of its largest entry).

    python tools/kernel_ab.py [c2] [c3] [c5] [m134] [--reps 12] [--variants 'soa;pull;ell;ell:RB=12']

A variant is `layout[:ENV=VALUE,...]` with ENV short names RB (MDE_B200_TILE_RB), STILE (MDE_B200_STILE_MB).
Prints one JSON line per (workload, variant)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench
import pymde_b200 as pm
from pymde_b200 import _lib

dev = torch.device("cuda", 0)
lib = _lib.load()
PEAK = 6569.3
try:
    PEAK = float(json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
SHORT = {"RB": "MDE_B200_TILE_RB", "STILE": "MDE_B200_STILE_MB", "MIN": "MDE_B200_TILE_MIN", "EPL": "MDE_B200_PULL_EPL",
         "REP": "MDE_B200_PULL_REP"}
flush = None


def set_variant(v):
    for k in list(SHORT.values()) + ["MDE_B200_LAYOUT"]:
        os.environ.pop(k, None)
    lay, _, rest = v.partition(":")
    os.environ["MDE_B200_LAYOUT"] = lay
    for kv in filter(None, rest.split(",")):
        k, val = kv.split("=")
        os.environ[SHORT[k]] = val


def time_kernel(mde, X, reps, cold=True):
    global flush
    lay = mde._layout()
    st = torch.cuda.current_stream(dev).cuda_stream
    g = torch.zeros_like(X)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    if flush is None:
        flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    ts = []
    for it in range(reps + 3):
        if cold:
            flush.fill_(it & 0xFF)
        g.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(lib.mde_distortion(lay.handle, X.data_ptr(), X.shape[1], g.data_ptr(), None, st))
        b.record()
        torch.cuda.synchronize()
        if it >= 3:
            ts.append(a.elapsed_time(b))
    g.zero_()
    loss.zero_()
    _lib.check(lib.mde_distortion(lay.handle, X.data_ptr(), X.shape[1], g.data_ptr(), loss.data_ptr(), st))
    torch.cuda.synchronize()
    return float(np.median(ts)), float(np.min(ts)), float(loss.item()), g


def run(name, n, m, edges, make_f, variants, reps, k=1):
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
    X = torch.randn(n, m, device=dev, generator=gen)
    X -= X.mean(0)
    p = edges.shape[0]
    b_alg = p * (8 + 4 * k) + 2 * n * m * 4 + 8
    ref = None
    for v in variants:
        set_variant(v)
        try:
            mde = pm.MDE(n, m, edges, make_f(), pm.Centered(), device=dev)
            med, mn, loss, g = time_kernel(mde, X, reps)
            warm, _, _, _ = time_kernel(mde, X, max(4, reps // 2), cold=False)
        except Exception as ex:  # keep going: one broken variant must not hide the others
            print(json.dumps({"workload": name, "variant": v, "error": repr(ex)[:300]}), flush=True)
            continue
        out = {"workload": name, "variant": v, "n": n, "m": m, "p": p, "kernel_us_cold_median": med * 1e3,
               "kernel_us_cold_min": mn * 1e3, "kernel_us_warm_median": warm * 1e3,
               "frac_cold": b_alg / (med * 1e-3) / 1e9 / PEAK, "loss_sum": loss,
               "layout_mb": lib.mde_edges_nbytes(mde._layout().handle) / 1e6}
        if ref is None:
            ref = (loss, g.clone())
        else:
            out["loss_rel_diff_vs_first"] = abs(loss - ref[0]) / abs(ref[0])
            out["grad_max_diff_over_max"] = float((g - ref[1]).abs().max() / ref[1].abs().max())
        print(json.dumps(out), flush=True)
        del mde, g
        torch.cuda.empty_cache()


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    reps = 12
    variants = ["soa", "tiles"]
    for i, a in enumerate(sys.argv):
        if a == "--reps":
            reps = int(sys.argv[i + 1])
        if a == "--variants":
            variants = sys.argv[i + 1].split(";")
    args = [a for a in args if not a.isdigit() and ";" not in a and a not in variants]
    which = args or ["c2"]
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    if "c2" in which:
        edges, w = bench.c2_edges(0)
        wt = torch.tensor(w, device=dev)
        run("C2", bench.N_ITEMS, 2, torch.tensor(edges, device=dev),
            lambda: pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log), variants, reps)
    if "m134" in which:
        n, p = 50000, 1_000_000
        e = torch.randint(0, n, (p, 2), device=dev, generator=g)
        e = e[e[:, 0] != e[:, 1]]
        w = torch.where(torch.rand(e.shape[0], device=dev, generator=g) < 0.5, 1.0, -1.0)
        dl = torch.rand(e.shape[0], device=dev, generator=g) * 3 + 0.5
        for m in (1, 3, 4):
            run("m%d pushpull" % m, n, m, e, lambda: pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log),
                variants, 4)
            run("m%d huber" % m, n, m, e, lambda: pm.losses.Huber(dl, 0.5), variants, 4)
    if "c3" in which:
        n, p = 44682, 20_000_000
        e = torch.randint(0, n, (p, 2), device=dev, generator=g)
        e = e[e[:, 0] != e[:, 1]]
        delta = torch.randint(1, 9, (e.shape[0],), device=dev, generator=g).float() * 0.25
        run("C3-shaped (n=44682, 2e7 pairs, losses.Huber)", n, 2, e, lambda: pm.losses.Huber(delta, 0.5), variants, 6)
        del e, delta
    if "c5" in which:
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        import bench_scale
        n, p = 10_000_000, 100_000_000
        e, w = bench_scale.sbm_edges(n, p, 1000, dev)
        run("C5-shaped (SBM n=1e7, 1e8 edges)", n, 2, e,
            lambda: pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log), variants, 5)


if __name__ == "__main__":
    main()
