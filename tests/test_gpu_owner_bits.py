"""The owner pass computes fixed bits: sha1 digests of the gradient, and the fp64 loss sum, recorded on an H100 from the
build before the kernel's loads were reorganised (tests/golden/owner_bits.json, written by
tests/golden/make_owner_bits_golden.py).  The entry order per lane, the __fadd_rn accumulation, the shuffle tree and
the per-thread fp64 loss order fix every bit, so a change to how the kernel fetches its operands must reproduce them.

Cases: the C2 slice generator (n = 20 000, m = 2) on the MUFU kernel and with MDE_B200_KERNEL=precise; the hub graph of
test_gpu_owner_pass (degree 5 200 hub, isolated and coincident rows, duplicate edges) at m = 1..4 with PushAndPull and
Huber; the same graph with caller-supplied coefficients (mde_scatter_external)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import bench
from tests.test_gpu_owner_pass import _exact_graph

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "owner_bits.json")
_ENV = ("MDE_B200_LAYOUT", "MDE_B200_KERNEL", "MDE_B200_DETERMINISTIC")

CASES = (["c2slice-fast", "c2slice-precise"] + ["hub-pushpull-m%d" % m for m in (1, 2, 3, 4)] +
         ["hub-huber-m%d" % m for m in (1, 2, 3, 4)] + ["hub-external-m%d" % m for m in (1, 2, 3, 4)])


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


@pytest.fixture(scope="module")
def recorded():
    with open(GOLDEN) as fh:
        return json.load(fh)


def evaluate(case):
    """{"grad_sha1": ..., "loss_hex": ...} of `case` on the library as built (kind-0 layout, owner kernel)."""
    import pymde_b200 as pm
    from pymde_b200 import _lib, util
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    kind, fn, tail = case.split("-")[0], case.split("-")[1], case.split("-")[-1]
    gext = None
    if kind == "c2slice":
        n, m = 20000, 2
        edges, w = bench.c2_edges(0, n=n, k=15)
        X = bench.initial_iterate(1, n=n, m=m)
        if fn == "precise":
            os.environ["MDE_B200_KERNEL"] = "precise"
        f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
    else:
        n, m = 6000, int(tail[1:])
        edges, g, w, X4, _ = _exact_graph(200 + m, n)
        # quarter-integer rows keep the coincident pairs (d = 0); the irrational factor makes the sums inexact
        X = np.ascontiguousarray(X4[:, :m] * np.float32(0.25 * np.sqrt(2.0)))
        if fn == "huber":
            f = pm.losses.Huber(torch.tensor(np.abs(g) + 0.5, device=dev), 0.5)
        else:
            f = pm.penalties.PushAndPull(torch.tensor(w, device=dev), pm.penalties.Log1p, pm.penalties.Log)
        if fn == "external":
            gext = torch.tensor(np.random.default_rng(7).standard_normal(len(edges)).astype(np.float32), device=dev)
    try:
        mde = pm.MDE(n, m, torch.tensor(edges, device=dev), f, pm.Centered(), device=dev)
        lay = mde._layout()
    finally:
        os.environ.pop("MDE_B200_KERNEL", None)
    assert int(lib.mde_edges_kind(lay.handle)) == 0
    Xd = torch.tensor(X, device=dev)
    grad = torch.zeros_like(Xd)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    if gext is not None:
        _lib.check(lib.mde_scatter_external(lay.handle, Xd.data_ptr(), m, gext.data_ptr(), grad.data_ptr(),
                                            util.stream_ptr(dev)))
    else:
        _lib.check(lib.mde_distortion(lay.handle, Xd.data_ptr(), m, grad.data_ptr(), loss.data_ptr(),
                                      util.stream_ptr(dev)))
    torch.cuda.synchronize()
    assert torch.isfinite(grad).all() and bool(grad.abs().max() > 0)
    return {"grad_sha1": hashlib.sha1(grad.cpu().numpy().tobytes()).hexdigest(), "loss_hex": float(loss.item()).hex()}


def test_fixture_lists_every_case(recorded):
    assert sorted(recorded["cases"]) == sorted(CASES)
    assert "H100" in recorded["gpu"]


@gpu
@pytest.mark.parametrize("case", CASES)
def test_owner_pass_reproduces_the_recorded_bits(case, recorded):
    assert evaluate(case) == recorded["cases"][case]
