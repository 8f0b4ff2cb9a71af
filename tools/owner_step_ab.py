#!/usr/bin/env python
"""A/B of two (or more) builds of libmde_b200.so on the benchmark's solver step and on the owner kernel alone.

    python tools/owner_step_ab.py [--libs BASE.so NEW.so ...] [--pairs 3] [--quick] [--out DIR]

The first library is the base (default `_ab/libmde_base.so`, a build of the parent commit), the others are compared
against it (default: the tree's own `pymde_b200/libmde_b200.so`).  Every arm runs in a subprocess of its own, which
points `pymde_b200._lib.LIB_PATH` at its library before `load()`; the arms alternate, `--pairs` rounds.  The workload
is bench.py's (C2: `bench.c2_edges(0)`, `bench.initial_iterate(0)`), taken by import.

Per arm and round, one JSON line:
  gpu                  card name, power limit, max SM clock, read in the same process
  step_us              solver step: warm-up, then 5 windows of 100 steps between CUDA events, median (and all five)
  owner_warm_us        mde_distortion alone, X and layout L2-resident: 200 launches between two events
  owner_cold_us        mde_distortion alone, 512 MB flush before each launch (as bench.kernel_roofline), mean of 20
  l2_read_25mb_us      a plain float4 read of a 25 MB L2-resident buffer (torch sum), 200 launches between two events:
                       what "L2 bandwidth" is on this card on that day
  split_us             (first round) head / vec / owner kernel time per step, torch.profiler CUDA activities in a run
                       of its own
  m134                 (first round) warm kernel time and solver step (3 windows of 100 steps) on the m = 1, 3, 4
                       shapes of kernel_ab.py (Huber, PushAndPull)
and an .npz with the raw results: gradient and loss sum at X0, embedding and statistics after the timed steps, and
the m134 gradients.  The parent compares every arm with the base byte for byte (`np.array_equal` on the raw bytes)
and prints the verdict and the spread of each arm.

`--quick` rehearses at a tiny size.  There is no CPU path: without a CUDA device the tool stops with an error after
the host-side set-up."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
import bench  # noqa: E402

WINDOWS, WINDOW_STEPS, WARMUP = 5, 100, 10


def workload(quick):
    n = 3000 if quick else bench.N_ITEMS
    edges, w = bench.c2_edges(0, n=n) if quick else bench.c2_edges(0)
    X0 = bench.initial_iterate(0, n=n) if quick else bench.initial_iterate(0)
    return n, edges, w, X0


# ------------------------------------------------------------------------------------------
# one arm (subprocess)
# ------------------------------------------------------------------------------------------
def between_events(torch, fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def kernel_split(torch, solver, steps):
    """Per-step device time of the three kernels of a solver step, from a profiled run of `steps` steps."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        solver.run(steps)
        torch.cuda.synchronize()
    out = {"head": 0.0, "vec": 0.0, "owner": 0.0, "other": 0.0}
    names = {"step_head_kernel": "head", "step_vec_kernel": "vec", "distortion_owner_kernel": "owner"}
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", None)
        if t is None:
            t = getattr(ev, "self_cuda_time_total", 0.0)
        key = next((v for k, v in names.items() if k in ev.key), "other")
        out[key] += float(t) / steps
    return out


def worker(args):
    import torch
    import pymde_b200 as pm
    from pymde_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(args.worker)
    lib = _lib.load()
    if not torch.cuda.is_available():
        raise SystemExit("owner_step_ab: no CUDA device; nothing here is measured on the CPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    n, edges, w, X0 = workload(args.quick)
    m = bench.EMBED_DIM
    wt = torch.tensor(w, device=dev)
    f = pm.penalties.PushAndPull(wt, pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, m, torch.tensor(edges, device=dev), f, pm.Centered(), device=dev)
    X0d = torch.tensor(X0, device=dev)
    lay = mde._layout()
    res = {"lib": args.worker, "round": args.round, "gpu": bench.gpu_identity(dev), "n": n, "p": int(len(edges)),
           "layout_kind": int(lib.mde_edges_kind(lay.handle))}
    raw = {}

    # gradient and loss at X0
    g = torch.zeros_like(X0d)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    _lib.check(lib.mde_distortion(lay.handle, X0d.data_ptr(), m, g.data_ptr(), loss.data_ptr(), st))
    torch.cuda.synchronize()
    raw["grad_x0"], raw["loss_x0"] = g.cpu().numpy(), loss.cpu().numpy()

    # the solver step, as bench.py times it
    total = WARMUP + WINDOWS * WINDOW_STEPS
    solver = mde._solver(mde.constraint, 10, total + 8)
    solver.begin(X0d, 0.0)
    solver.run(WARMUP)
    torch.cuda.synchronize()
    steps = [WINDOW_STEPS] * WINDOWS
    windows, done = bench.timed_windows(solver, steps, torch.cuda.synchronize, torch, dev, 1)
    per = [ms * 1e3 / k for ms, k in zip(windows, steps)]
    res["step_us"], res["step_us_windows"] = float(np.median(per)), per
    avg, rn, pct, stp, fe = solver.stats(done)
    raw["embedding"] = solver.x_view().cpu().numpy()
    raw["average_distortions"], raw["residual_norms"] = np.asarray(avg), np.asarray(rn)
    raw["step_size_percents"], raw["step_sizes"] = np.asarray(pct), np.asarray(stp)
    Xw = solver.x_view().clone()  # a mid-solve iterate: what the kernel sees in the timed steps

    # the owner kernel alone: warm, cold, and the L2 read ceiling
    def launch():
        _lib.check(lib.mde_distortion(lay.handle, Xw.data_ptr(), m, g.data_ptr(), None, st))
    for _ in range(20):
        launch()
    res["owner_warm_us"] = [between_events(torch, launch, 200) for _ in range(3)]
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    cold = []
    for it in range(24):
        flush.fill_(it & 0xFF)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        launch()
        b.record()
        torch.cuda.synchronize()
        if it >= 4:
            cold.append(a.elapsed_time(b) * 1e3)
    res["owner_cold_us"] = float(np.mean(cold))
    del flush
    buf = torch.ones((25 << 20) // 16, 4, device=dev)
    for _ in range(20):
        buf.sum()
    res["l2_read_25mb_us"] = [between_events(torch, buf.sum, 200) for _ in range(3)]
    res["l2_read_25mb_gbs"] = buf.numel() * 4 / (min(res["l2_read_25mb_us"]) * 1e-6) / 1e9

    if args.round == 0:
        s2 = mde._solver(mde.constraint, 10, 200 + 8)
        s2.begin(X0d, 0.0)
        s2.run(WARMUP)
        res["split_us"] = kernel_split(torch, s2, 100)
        res["m134"] = m134(torch, pm, _lib, lib, dev, st, raw, args.quick)

    np.savez(args.raw, **raw)
    print("ARM " + json.dumps(res), flush=True)


def m134(torch, pm, _lib, lib, dev, st, raw, quick):
    """The m = 1, 3, 4 shapes of kernel_ab.py on the default layout: the other owner-kernel instantiations."""
    n, p = (2000, 40000) if quick else (50000, 1_000_000)
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    e = torch.randint(0, n, (p, 2), device=dev, generator=gen)
    e = e[e[:, 0] != e[:, 1]]
    w = torch.where(torch.rand(e.shape[0], device=dev, generator=gen) < 0.5, 1.0, -1.0)
    dl = torch.rand(e.shape[0], device=dev, generator=gen) * 3 + 0.5
    out = {}
    for m in (1, 3, 4):
        X = torch.randn(n, m, device=dev, generator=gen)
        X -= X.mean(0)
        for name, fn in (("pushpull", lambda: pm.penalties.PushAndPull(w, pm.penalties.Log1p, pm.penalties.Log)),
                         ("huber", lambda: pm.losses.Huber(dl, 0.5))):
            mde = pm.MDE(n, m, e, fn(), pm.Centered(), device=dev)
            lay = mde._layout()
            g = torch.zeros_like(X)
            loss = torch.zeros(1, dtype=torch.float64, device=dev)
            _lib.check(lib.mde_distortion(lay.handle, X.data_ptr(), m, g.data_ptr(), loss.data_ptr(), st))
            torch.cuda.synchronize()
            raw["m%d_%s_grad" % (m, name)], raw["m%d_%s_loss" % (m, name)] = g.cpu().numpy(), loss.cpu().numpy()

            def launch():
                _lib.check(lib.mde_distortion(lay.handle, X.data_ptr(), m, g.data_ptr(), None, st))
            for _ in range(10):
                launch()
            row = {"kind": int(lib.mde_edges_kind(lay.handle)), "warm_us": between_events(torch, launch, 100)}
            solver = mde._solver(mde.constraint, 10, WARMUP + 3 * WINDOW_STEPS + 8)
            solver.begin(X, 0.0)
            solver.run(WARMUP)
            ws, done = bench.timed_windows(solver, [WINDOW_STEPS] * 3, torch.cuda.synchronize, torch, dev, 1)
            row["step_us"] = float(np.median(ws)) * 1e3 / WINDOW_STEPS
            raw["m%d_%s_embedding" % (m, name)] = solver.x_view().cpu().numpy()
            out["m%d %s" % (m, name)] = row
    return out


# ------------------------------------------------------------------------------------------
# parent
# ------------------------------------------------------------------------------------------
def same_bytes(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=[os.path.join(REPO, "_ab", "libmde_base.so"),
                                                  os.path.join(REPO, "pymde_b200", "libmde_b200.so")])
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the arms' JSON lines (ab.jsonl)")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--round", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--raw", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)

    if args.pairs < 3 and not args.quick:
        ap.error("--pairs must be at least 3")
    for lib in args.libs:
        if not os.path.exists(lib):
            raise SystemExit("owner_step_ab: no library at %s (build the parent commit there)" % lib)
    n, edges, w, X0 = workload(args.quick)
    print("workload: n=%d p=%d m=%d, %d arms x %d rounds" % (n, len(edges), bench.EMBED_DIM, len(args.libs), args.pairs),
          flush=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("owner_step_ab: no CUDA device; nothing here is measured on the CPU")

    tmp = tempfile.mkdtemp(prefix="owner_step_ab_")
    arms = {lib: [] for lib in args.libs}
    raws = {}
    for r in range(args.pairs):
        for k, lib in enumerate(args.libs):
            rawf = os.path.join(tmp, "arm%d_round%d.npz" % (k, r))
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", lib, "--round", str(r), "--raw", rawf]
            out = subprocess.run(cmd + (["--quick"] if args.quick else []), capture_output=True, text=True)
            line = next((ln[4:] for ln in out.stdout.splitlines() if ln.startswith("ARM ")), None)
            if out.returncode != 0 or line is None:
                raise SystemExit("owner_step_ab: arm %s failed\n%s\n%s" % (lib, out.stdout[-2000:], out.stderr[-4000:]))
            print(line, flush=True)
            arms[lib].append(json.loads(line))
            raws[(lib, r)] = dict(np.load(rawf))

    base = args.libs[0]
    verdict = {"base": base, "arms": []}
    for lib in args.libs:
        rs = arms[lib]
        steps = [a["step_us"] for a in rs]
        warm = [min(a["owner_warm_us"]) for a in rs]
        row = {"lib": lib, "step_us": steps, "step_us_median": float(np.median(steps)),
               "step_us_spread": max(steps) - min(steps), "owner_warm_us_median": float(np.median(warm)),
               "owner_cold_us_median": float(np.median([a["owner_cold_us"] for a in rs])),
               "l2_read_25mb_us_min": min(min(a["l2_read_25mb_us"]) for a in rs),
               "split_us": rs[0].get("split_us")}
        diff = sorted({k for r in range(args.pairs) for k in raws[(base, 0)]
                       if k in raws[(lib, r)] and not same_bytes(raws[(base, 0)][k], raws[(lib, r)][k])})
        row["byte_identical_to_base"] = not diff
        row["differing"] = diff
        if lib != base:
            bs = [a["step_us"] for a in arms[base]]
            row["slowest_below_fastest_base"] = max(steps) < min(bs)
            row["median_gain_percent"] = 100.0 * (1.0 - np.median(steps) / np.median(bs))
        verdict["arms"].append(row)
    print("VERDICT " + json.dumps(verdict), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab.jsonl"), "w") as fh:
            for lib in args.libs:
                for a in arms[lib]:
                    fh.write(json.dumps(a) + "\n")
            fh.write(json.dumps(verdict) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
