"""Two GPUs, one process each (self-skips on a box with fewer): the edge-sharded evaluation and solve of
pymde_b200/dist.py against the C oracle and the single-GPU solve -- peer-memory all-reduce kernels
(mde_solver.cu::allreduce_kernel and allreduce_push_kernel) and the NCCL host hook.  The worker is tests/mgpu_worker.py."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


@pytest.mark.gpu
def test_two_rank_sharded_evaluation_and_solve():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(REPO, "tests", "mgpu_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=REPO)
    lines = [l for l in out.stdout.splitlines() if l.startswith("MGPU_RESULT ")]
    assert out.returncode == 0 and lines, (out.stdout[-2000:], out.stderr[-4000:])
    r = json.loads(lines[-1][len("MGPU_RESULT "):])
    # (i) sharded evaluation == oracle on the whole edge list (north_star: 1e-5 relative on the value)
    assert r["eval_value_rel"] < 1e-5
    assert r["eval_grad_err"] < 3e-5
    for transport in ("peer", "nccl"):
        t = r[transport]
        assert t["iterations"] == 25 and t["x_identical"] and t["decreased"]
        assert t["loss0_rel"] < 1e-5 and t["resid0_rel"] < 1e-4
        assert t["first3_rel_vs_single"] < 1e-3
    assert r["peer"]["peer_memory"] and not r["nccl"]["peer_memory"]
    # (iv) gradient above the one-shot limit: write-based all-reduce
    t = r["big"]["push"]
    assert t["iterations"] == 8 and t["x_identical"] and t["decreased"]
    assert t["loss0_rel"] < 1e-5 and t["resid0_rel"] < 1e-4
    assert t["first3_rel_vs_single"] < 1e-3
    # (v) non-fused sharded problem (external callable -> host-stepped solver): global objective, identical replicas
    assert r["generic"]["value_rel"] < 1e-5 and r["generic"]["x_identical"] and r["generic"]["decreased"]
    # (iii) converged problem: the north_star's criterion
    c = r["converged"]
    assert c["x_identical"] and c["iterations"] < 800 and c["single_iterations"] < 800
    assert c["rel"] < 1e-5
