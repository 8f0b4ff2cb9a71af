#!/usr/bin/env python
"""Worker of tests/test_gpu_multi.py (run under torch.distributed.run, one rank per GPU).

Every rank builds its shard of the SAME problem (pymde_b200.dist.shard_mde) and checks
  (i)   the sharded evaluation (value AND gradient through autograd) against the C oracle on the whole edge list,
  (ii)  the sharded solve, peer-memory all-reduce (graph-captured) AND the NCCL host hook: iteration-0 loss and
        gradient norm against the oracle, first iterations against the single-GPU solve, bit-identical X on all ranks,
  (iii) a converged problem (quadratic penalties, Standardized): final average distortion within 1e-5 of the
        single-GPU solve.
Prints one JSON line `MGPU_RESULT {...}` on rank 0."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.distributed as td
import bench
import pymde_b200 as pm
from pymde_b200 import dist as pdist
from oracle import c_oracle, mde_oracle as O

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr); dev = torch.device("cuda", lr)
td.init_process_group("nccl", device_id=dev)
res = {"world": world}
n, m = 20000, 2
edges, w = bench.c2_edges(0, n=n, k=10)
X0 = bench.initial_iterate(0, n=n, m=m)
et, wt = torch.tensor(edges), torch.tensor(w)
mk = lambda lo, hi: pm.penalties.PushAndPull(wt[lo:hi].to(dev), pm.penalties.Log1p, pm.penalties.Log)
spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
v_ref, g_ref = c_oracle.average_distortion(X0, edges, spec, True)
r_ref = float(np.sqrt((g_ref ** 2).sum()))


def digests_equal(X):
    import hashlib
    d = hashlib.sha1(X.detach().cpu().numpy().tobytes()).hexdigest()
    out = [None] * world
    td.all_gather_object(out, d)
    return len(set(out)) == 1


# (i) evaluation outside the solver
mde = pdist.shard_mde(pm.MDE, n, m, et, mk, pm.Centered(), dev, transport="peer")
Xg = torch.tensor(X0, device=dev, requires_grad=True)
v = mde.average_distortion(Xg)
v.backward()
res["eval_value_rel"] = abs(v.item() - v_ref) / abs(v_ref)
res["eval_grad_err"] = float(np.abs(Xg.grad.cpu().numpy() - g_ref).max() / np.abs(g_ref).max())

# (ii) solves
K = 25
full_stats = None
if rank == 0:
    full = pm.MDE(n, m, et.to(dev), mk(0, len(edges)), pm.Centered(), device=dev)
    full.embed(X=torch.tensor(X0, device=dev), max_iter=K, eps=0.0)
    full_stats = np.array(full.solve_stats.average_distortions)
for transport in ("peer", "nccl"):
    md = pdist.shard_mde(pm.MDE, n, m, et, mk, pm.Centered(), dev, transport=transport)
    X = md.embed(X=torch.tensor(X0, device=dev), max_iter=K, eps=0.0)
    st = md.solve_stats
    a = np.array(st.average_distortions)
    r = {"iterations": st.iterations, "x_identical": digests_equal(X),
         "loss0_rel": abs(a[0] - v_ref) / abs(v_ref), "resid0_rel": abs(st.residual_norms[0] - r_ref) / r_ref,
         "decreased": bool(a[-1] < 0.5 * a[0]),
         "peer_memory": bool(md.__dict__["_device_solver"][1].peer_memory)}
    if rank == 0:
        r["first3_rel_vs_single"] = float(np.abs(a[:3] - full_stats[:3]).max() / np.abs(full_stats[:3]).max())
        r["final_rel_vs_single"] = float(abs(a[-1] - full_stats[-1]) / abs(full_stats[-1]))
    res[transport] = r
    del md

# (iii) a problem that converges: final value must agree to 1e-5
rng = np.random.default_rng(1)
n2, p2 = 3000, 30000
e2 = rng.integers(0, n2, (p2 * 2, 2)); e2 = e2[e2[:, 0] != e2[:, 1]][:p2]
w2 = (rng.random(p2).astype(np.float32) + 0.5)
e2t, w2t = torch.tensor(e2), torch.tensor(w2)
mk2 = lambda lo, hi: pm.penalties.Quadratic(w2t[lo:hi].to(dev))
gen = torch.Generator(); gen.manual_seed(0)
X2 = pm.Standardized().initialization(n2, 2, dev) if False else None
Xi = torch.randn(n2, 2, generator=gen).to(dev)
Xi = pm.Standardized().project_onto_constraint(Xi, inplace=True)
ms = pdist.shard_mde(pm.MDE, n2, 2, e2t, mk2, pm.Standardized(), dev, transport="peer")
ms.embed(X=Xi, max_iter=800, eps=1e-5)
conv = {"iterations": ms.solve_stats.iterations, "value": float(ms.solve_stats.average_distortions[-1]),
        "residual": float(ms.solve_stats.residual_norms[-1]), "x_identical": digests_equal(ms.X)}
if rank == 0:
    one = pm.MDE(n2, 2, e2t.to(dev), mk2(0, p2), pm.Standardized(), device=dev)
    one.embed(X=Xi, max_iter=800, eps=1e-5)
    conv["single_value"] = float(one.solve_stats.average_distortions[-1])
    conv["single_iterations"] = one.solve_stats.iterations
    conv["rel"] = abs(conv["value"] - conv["single_value"]) / abs(conv["single_value"])
res["converged"] = conv

# (iv) a gradient above 4 MB (n = 600 000): the write-based ("push") all-reduce
n3 = 600_000
e3, w3 = bench.c5_shard(3, n=n3, p=3_000_000, block=5_000)
X3 = bench.initial_iterate(4, n3, 2)
e3t, w3t = torch.tensor(e3), torch.tensor(w3)
mk3 = lambda lo, hi: pm.penalties.PushAndPull(w3t[lo:hi].to(dev), pm.penalties.Log1p, pm.penalties.Log)
spec3 = O.FnSpec(O.P_LOG1P, w3, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
v3_ref, g3_ref = c_oracle.average_distortion(X3, e3, spec3, True)
r3_ref = float(np.sqrt((g3_ref ** 2).sum()))
one3 = None
if rank == 0:
    one = pm.MDE(n3, 2, e3t.to(dev), mk3(0, len(e3)), pm.Centered(), device=dev)
    one.embed(X=torch.tensor(X3, device=dev), max_iter=8, eps=0.0)
    one3 = np.array(one.solve_stats.average_distortions)
    del one
mb = pdist.shard_mde(pm.MDE, n3, 2, e3t, mk3, pm.Centered(), dev, transport="peer")
Xb = mb.embed(X=torch.tensor(X3, device=dev), max_iter=8, eps=0.0)
sb = mb.solve_stats
ab = np.array(sb.average_distortions)
rb = {"iterations": sb.iterations, "x_identical": digests_equal(Xb), "loss0_rel": abs(ab[0] - v3_ref) / abs(v3_ref),
      "resid0_rel": abs(sb.residual_norms[0] - r3_ref) / r3_ref, "decreased": bool(ab[-1] < ab[0])}
if rank == 0:
    rb["first3_rel_vs_single"] = float(np.abs(ab[:3] - one3[:3]).max() / np.abs(one3[:3]).max())
del mb
res["big"] = {"push": rb}

# (v) a sharded problem the device solver does not take (arbitrary callable): the host-stepped solver must still see
#     the GLOBAL objective (EdgeLayout all-reduces evaluations), so the replicas stay identical
wq = torch.rand(len(edges), generator=torch.Generator().manual_seed(5)) + 0.5
lo, hi = pdist.shard_range(len(edges), rank, world)
wloc = wq[lo:hi].to(dev)
mg = pm.MDE(n, m, et[lo:hi].to(dev), lambda d: wloc * d ** 2, pm.Centered(), device=dev)
pdist.attach(mg, rank, world, len(edges), dev)
Xg0 = torch.tensor(X0, device=dev)
vg = mg.average_distortion(Xg0).item()
vg_ref = float((wq.double().numpy() * (np.linalg.norm(X0[edges[:, 0]].astype(np.float64) - X0[edges[:, 1]], axis=1) ** 2)).mean())
Xg = mg.embed(X=Xg0, max_iter=6, eps=0.0)
res["generic"] = {"value_rel": abs(vg - vg_ref) / abs(vg_ref), "x_identical": digests_equal(Xg),
                  "decreased": bool(mg.solve_stats.average_distortions[-1] < mg.solve_stats.average_distortions[0])}
if rank == 0:
    print("MGPU_RESULT " + json.dumps(res), flush=True)
td.barrier()
td.destroy_process_group()
