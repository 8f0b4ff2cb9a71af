"""GPU parity tests: the CUDA kernels (called through the C ABI via pymde_b200) against
(i) fixtures produced by the unmodified reference (tests/golden/*.npz), (ii) the numpy oracle on
seeded inputs, (iii) the reference's own known-answer tests.  Tolerances: fp32 arithmetic, so
1e-5 relative on values (north_star) and a scaled absolute tolerance on gradients."""
import numpy as np
import pytest
import torch

from oracle import mde_oracle as O
from tests.golden_cases import CASES, spec_for

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["auto", "soa", "tiles", "pull", "ell"], autouse=True)
def edge_layout(request, monkeypatch):
    """Every test of this file runs on each edge layout / kernel family: the library's own choice, the sorted-SoA
    layout (owner / quad / wide kernels), tile records (push kernel), pull records and ELL pull records
    (mde_edges.cuh).  Layouts that
    do not apply (m > 4, WeightedQuadratic's second array) fall back to SoA inside the library."""
    if request.param != "auto":
        monkeypatch.setenv("MDE_B200_LAYOUT", request.param)
    else:
        monkeypatch.delenv("MDE_B200_LAYOUT", raising=False)
    return request.param


def _pm():
    import pymde_b200 as pm
    return pm


def make_function(pm, name, fg, tag="f32", device="cuda"):
    par0 = torch.tensor(fg["%s/%s/par0" % (name, tag)], dtype=torch.float32, device=device)
    pen, los = pm.penalties, pm.losses
    table = {
        "pen_linear": lambda: pen.Linear(par0),
        "pen_quadratic": lambda: pen.Quadratic(par0),
        "pen_cubic": lambda: pen.Cubic(par0),
        "pen_power_2.5": lambda: pen.Power(par0, 2.5),
        "pen_huber_0.5": lambda: pen.Huber(par0, 0.5),
        "pen_logistic_0.3_3": lambda: pen.Logistic(par0, 0.3, 3.0),
        "pen_log1p_1.5": lambda: pen.Log1p(par0, 1.5),
        "pen_log_1": lambda: pen.Log(par0, 1.0),
        "pen_invpower_1": lambda: pen.InvPower(par0, 1),
        "pen_logratio_2": lambda: pen.LogRatio(par0, 2),
        "pen_pushpull_log1p_log": lambda: pen.PushAndPull(par0, pen.Log1p, pen.Log),
        "pen_pushpull_default": lambda: pen.PushAndPull(par0),
        "pen_pushpull_quad_invpower": lambda: pen.PushAndPull(par0, pen.Quadratic, pen.InvPower),
        "loss_absolute": lambda: los.Absolute(par0),
        "loss_quadratic": lambda: los.Quadratic(par0),
        "loss_weighted_quadratic": lambda: los.WeightedQuadratic(par0),
        "loss_weighted_quadratic_w": lambda: los.WeightedQuadratic(
            par0, torch.tensor(fg["%s/%s/par1" % (name, tag)], dtype=torch.float32, device=device)),
        "loss_huber_0.7": lambda: los.Huber(par0, 0.7),
        "loss_cubic": lambda: los.Cubic(par0),
        "loss_power_1.5": lambda: los.Power(par0, 1.5),
        "loss_logistic": lambda: los.Logistic(par0),
        "loss_fractional": lambda: los.Fractional(par0),
        "loss_soft_fractional_10": lambda: los.SoftFractional(par0, 10.0),
    }
    return table[name]()


@pytest.mark.parametrize("name", sorted(CASES))
def test_function_eval_matches_reference(golden, name):
    pm = _pm()
    g = golden["functions"]
    f = make_function(pm, name, g)
    d = torch.tensor(g["%s/f32/d" % name], device="cuda", requires_grad=True)
    val = f(d)
    val.sum().backward()
    np.testing.assert_allclose(val.detach().cpu().numpy(), g["%s/f32/f" % name], rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(d.grad.cpu().numpy(), g["%s/f32/fp" % name], rtol=2e-5, atol=2e-6)
    # and against the float64 reference run (closed forms, tighter truth)
    np.testing.assert_allclose(val.detach().cpu().numpy(), g["%s/f64/f" % name], rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize("key", ["m1", "m2", "m3", "m4", "m7", "m16", "m2_zero", "m3_zero"])
def test_average_distortion_matches_reference(golden, key):
    pm = _pm()
    g, fg = golden["evals"], golden["functions"]
    edges = torch.tensor(g[key + "/edges"], device="cuda")
    Xn = g[key + "/X"]
    n, m = Xn.shape
    for name in sorted(CASES):
        f = make_function(pm, name, fg)
        mde = pm.MDE(n, m, edges, f, pm.Centered())
        X = torch.tensor(Xn, device="cuda", requires_grad=True)
        v = mde.average_distortion(X)
        v.backward()
        rv, rg = g["%s/%s/f64/value" % (key, name)], g["%s/%s/f64/grad" % (key, name)]
        np.testing.assert_allclose(v.item(), rv, rtol=1e-5, atol=1e-6, equal_nan=True, err_msg=name)
        fin = np.isfinite(rg)
        scale = max(1.0, float(np.abs(rg[fin]).max())) if fin.any() else 1.0
        np.testing.assert_allclose(X.grad.cpu().numpy(), rg, rtol=3e-5, atol=3e-5 * scale, equal_nan=True,
                                   err_msg=name)
        # forward-only branch (average_distortion.py:64-65) gives the same value
        v2 = mde.average_distortion(X.detach())
        np.testing.assert_allclose(v2.item(), v.item(), rtol=1e-6, equal_nan=True)


def test_per_edge_outputs_in_caller_order(golden):
    pm = _pm()
    g, fg = golden["evals"], golden["functions"]
    edges = torch.tensor(g["m2/edges"], device="cuda")
    X = torch.tensor(g["m2/X"], device="cuda")
    for name in sorted(CASES):
        mde = pm.MDE(X.shape[0], 2, edges, make_function(pm, name, fg), pm.Centered())
        np.testing.assert_allclose(mde.distances(X).cpu().numpy(), g["m2/%s/distances" % name], rtol=1e-6)
        np.testing.assert_allclose(mde.distortions(X).cpu().numpy(), g["m2/%s/distortions" % name],
                                   rtol=2e-5, atol=2e-6, err_msg=name)
    pairs, dist = mde.high_distortion_pairs(X)
    assert bool((dist[:-1] >= dist[1:]).all())
    assert pairs.shape == edges.shape and pairs.dtype == torch.int64
    # the caller's int64 edge list is never mutated
    assert torch.equal(mde.edges.cpu(), torch.tensor(g["m2/edges"]))


def test_known_answer_62_over_3():
    # pymde/test_optim.py:75-93
    pm = _pm()
    edges = np.array([(0, 1), (0, 2), (1, 2)])
    mde = pm.MDE(3, 2, edges, pm.penalties.Quadratic(torch.tensor([1.0, 2.0, 3.0])), pm.Standardized())
    X = torch.tensor([[0.0, 0.0], [1.0, 1.0], [3.0, 3.0]], device="cuda")
    np.testing.assert_allclose(mde.average_distortion(X).item(), 62.0 / 3, rtol=1e-6)


def test_gradient_vs_dense_incidence_oracle():
    # pymde/test_optim.py:97-118 (oracle pymde/util.py:425-451)
    pm = _pm()
    torch.manual_seed(0)
    edges = np.array([(0, 1), (0, 2), (1, 2)])
    w = torch.tensor([1.0, 2.0, 3.0])
    mde = pm.MDE(3, 2, edges, pm.penalties.Quadratic(w), pm.Standardized())
    X = torch.randn((3, 2), device="cuda", requires_grad=True)
    mde.average_distortion(X).backward()
    A = np.array([[1, 1, 0], [-1, 0, 1], [0, -1, -1]], dtype=np.float64)
    Xn = X.detach().cpu().double().numpy()
    gk = 2 * w.numpy() / 3
    np.testing.assert_allclose(X.grad.cpu().numpy(), A @ (np.diag(gk) @ (A.T @ Xn)), rtol=1e-5, atol=1e-6)


def test_zero_distance_zero_gradient_and_differences_norms():
    # pymde/test_optim.py:22-71
    pm = _pm()
    torch.manual_seed(0)
    edges = np.array([(0, 1), (0, 2), (1, 2)])
    X = torch.randn((3, 3), device="cuda")
    mde = pm.MDE(3, 3, edges, pm.penalties.Quadratic(torch.ones(3)), pm.Standardized())
    diff = X[edges[:, 0]] - X[edges[:, 1]]
    np.testing.assert_allclose(mde.differences(X).cpu().numpy(), diff.cpu().numpy())
    np.testing.assert_allclose(mde.distances(X).cpu().numpy(), diff.norm(dim=1).cpu().numpy(), rtol=1e-6)
    for f in (pm.penalties.Quadratic(torch.ones(1)), pm.penalties.Linear(torch.ones(1)),
              pm.penalties.Log1p(torch.ones(1))):
        mde1 = pm.MDE(3, 3, np.array([(0, 1)]), f, pm.Standardized())
        Xo = torch.ones((3, 3), device="cuda", requires_grad=True)
        mde1.average_distortion(Xo).backward()
        assert float(Xo.grad.abs().max()) == 0.0


def test_self_edges_raise():
    # pymde/test_optim.py:157-170
    pm = _pm()
    edges = np.array([(0, 1), (0, 0), (0, 2), (1, 2), (1, 1)])
    with pytest.raises(ValueError, match=r"The edge list must not contain self edges.*"):
        pm.MDE(3, 3, edges, pm.penalties.Quadratic(torch.ones(edges.shape[0])), pm.Standardized())


def test_cpu_device_is_rejected_loudly():
    pm = _pm()
    with pytest.raises(ValueError, match="CUDA"):
        pm.MDE(3, 2, np.array([(0, 1)]), pm.penalties.Quadratic(torch.ones(1)), device="cpu")


@pytest.mark.parametrize("key", ["n2_m2", "n10_m3", "n100_m3", "n1000_m2", "n257_m5", "n300_m40"])
def test_projections_match_reference(golden, key):
    pm = _pm()
    g = golden["projections"]
    Z = torch.tensor(g[key + "/Z"], device="cuda")
    n, m = Z.shape
    C = pm.Centered().project_onto_constraint(Z.clone(), inplace=True)
    np.testing.assert_allclose(C.cpu().numpy(), g[key + "/centered"], atol=2e-6)
    if n <= m:  # de-meaned X is rank deficient: the polar factor is not unique (SVD-implementation defined)
        return
    Xs = pm.Standardized().project_onto_constraint(Z.clone(), inplace=True)
    np.testing.assert_allclose(Xs.cpu().numpy(), g[key + "/standardized"], atol=3e-4, rtol=1e-4)
    Xs64 = Xs.double()
    np.testing.assert_allclose((Xs64.T @ Xs64 / n).cpu().numpy(), np.eye(m), atol=1e-4)  # test_util.py:20-71
    if n > 2:
        np.testing.assert_allclose(Xs.mean(0).cpu().numpy(), 0, atol=1e-5)
    Xref = torch.tensor(g[key + "/standardized"], device="cuda")
    T = pm.Standardized().project_onto_tangent_space(Xref, torch.tensor(g[key + "/G"], device="cuda"), inplace=True)
    np.testing.assert_allclose(T.cpu().numpy(), g[key + "/tangent"], atol=5e-5, rtol=1e-4)


def test_proj_standardized_invariants_reference_shapes():
    # pymde/test_util.py:20-71 incl. (1000, 250)
    pm = _pm()
    torch.manual_seed(0)
    P = pm.util.proj_standardized(torch.eye(2, device="cuda"))
    np.testing.assert_allclose((P.T @ P / 2.0).cpu().numpy(), np.eye(2), atol=1e-5)
    for n, m in ((10, 3), (100, 3), (1000, 2), (1000, 3), (1000, 250)):
        X = torch.randn((n, m), device="cuda")
        P = pm.util.proj_standardized(X, demean=True)
        P64 = P.double()
        np.testing.assert_allclose((P64.T @ P64 / n).cpu().numpy(), np.eye(m), atol=1e-4)
        np.testing.assert_allclose(P.mean(0).cpu().numpy(), np.zeros(m), atol=1e-5)
    I = pm.Standardized().initialization(5, 3)
    np.testing.assert_allclose((I.T @ I / 5).cpu().numpy(), np.eye(3), atol=1e-4)  # test_optim.py:13-18


@pytest.mark.parametrize("n,m", [(500, 33), (3000, 64), (1000, 100), (20000, 128), (1000, 250), (5000, 256)])
def test_wide_standardized_projection_and_tangent_match_fp64(n, m):
    """32 < m <= 256 (csrc/mde_project_wide.cu) against the reference formulas in fp64: the retraction is
    sqrt(n) U V^T of the de-meaned matrix (pymde/util.py:129-171), the tangent projection Z - X (Z^T X) / n
    (pymde/constraints.py:186-192)."""
    pm = _pm()
    g = torch.Generator(device="cuda").manual_seed(n + m)
    X = torch.randn((n, m), generator=g, device="cuda") * (1.0 + torch.arange(m, device="cuda") / m) + 0.3
    P = pm.util.proj_standardized(X, demean=True)
    Xc = X.double() - X.double().mean(0)
    U, _, Vh = torch.linalg.svd(Xc, full_matrices=False)
    ref = (n ** 0.5) * U @ Vh
    np.testing.assert_allclose(P.cpu().numpy(), ref.cpu().numpy(), atol=5e-5, rtol=0)
    P64 = P.double()
    np.testing.assert_allclose((P64.T @ P64 / n).cpu().numpy(), np.eye(m), atol=1e-4)
    np.testing.assert_allclose(P.mean(0).cpu().numpy(), np.zeros(m), atol=1e-5)
    # a nearly standardized matrix (what the solver retracts at every trial): same check
    Q = pm.util.proj_standardized(P + 0.01 * torch.randn((n, m), generator=g, device="cuda"), demean=True)
    Q64 = Q.double()
    np.testing.assert_allclose((Q64.T @ Q64 / n).cpu().numpy(), np.eye(m), atol=1e-4)
    # tangent space
    Z = torch.randn((n, m), generator=g, device="cuda")
    T = pm.Standardized().project_onto_tangent_space(P, Z, inplace=False)
    Tref = Z.double() - P64 @ (Z.double().T @ P64) / n
    np.testing.assert_allclose(T.cpu().numpy(), Tref.cpu().numpy(), atol=2e-5, rtol=1e-5)


def _random_problem(n, p, m, rng, push_pull=True):
    i = rng.integers(0, n, 2 * p)
    j = rng.integers(0, n, 2 * p)
    keep = i != j
    e = np.stack([i[keep], j[keep]], 1)
    e = np.unique(np.sort(e, axis=1), axis=0)[:p]
    rng.shuffle(e)
    flip = rng.random(len(e)) < 0.5
    e[flip] = e[flip][:, ::-1]
    w = rng.choice([1.0, 2.0, -1.0], len(e)).astype(np.float32) if push_pull else \
        rng.uniform(0.5, 2.0, len(e)).astype(np.float32)
    X = rng.standard_normal((n, m)).astype(np.float32)
    return e.astype(np.int64), w, X


@pytest.mark.parametrize("m", [1, 2, 3, 4, 5, 8, 12, 16, 20, 33, 64, 100, 128, 200])
def test_fused_kernel_vs_oracle_all_widths(m):
    """Every kernel shape (thread-per-edge m<=4, group-per-edge 8/16/32 lanes, float4 and scalar
    columns) against the numpy oracle on a seeded random multigraph-free edge list."""
    pm = _pm()
    rng = np.random.default_rng(100 + m)
    n, p = 3000, 20000
    e, w, X = _random_problem(n, p, m, rng)
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    v_ref, g_ref = O.average_distortion(X.astype(np.float64), e, spec, True, np.float64)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(n, m, torch.tensor(e, device="cuda"), f)
    Xt = torch.tensor(X, device="cuda", requires_grad=True)
    v = mde.average_distortion(Xt)
    v.backward()
    np.testing.assert_allclose(v.item(), v_ref, rtol=1e-5)
    scale = float(np.abs(g_ref).max())
    np.testing.assert_allclose(Xt.grad.cpu().numpy(), g_ref, atol=2e-5 * scale, rtol=1e-4)
    d_ref, _ = O.edge_distances(X.astype(np.float64), e)
    np.testing.assert_allclose(mde.distances(Xt.detach()).cpu().numpy(), d_ref, rtol=1e-5)


def test_gradient_is_sum_zero_and_linear_in_weights():
    """Size-independent properties at a larger size: column sums of the gradient vanish
    (every edge contributes +c and -c), and E is linear in the weights."""
    pm = _pm()
    rng = np.random.default_rng(5)
    n, p, m = 200000, 3000000, 2
    e, w, X = _random_problem(n, p, m, rng, push_pull=False)
    et, Xt = torch.tensor(e, device="cuda"), torch.tensor(X, device="cuda")
    wt = torch.tensor(w, device="cuda")
    vals = []
    for scale in (1.0, 3.0):
        mde = pm.MDE(n, m, et, pm.penalties.Log1p(wt * scale))
        Xg = Xt.clone().requires_grad_(True)
        v = mde.average_distortion(Xg)
        v.backward()
        vals.append(v.item())
        gs = Xg.grad.double().sum(0).abs().max().item()
        assert gs < 1e-6 * float(Xg.grad.abs().max()) * n ** 0.5 + 1e-7
    np.testing.assert_allclose(vals[1], 3.0 * vals[0], rtol=2e-6)
    # against the oracle on a bounded sample of the same edges
    sub = slice(0, 200000)
    spec = O.FnSpec(O.P_LOG1P, w[sub], (1.5, 0, 0))
    v_ref, _ = O.average_distortion(X.astype(np.float64), e[sub], spec, False)
    mde = pm.MDE(n, m, et[sub], pm.penalties.Log1p(wt[sub]))
    np.testing.assert_allclose(mde.average_distortion(Xt).item(), v_ref, rtol=1e-5)


def test_external_callable_distortion_function():
    """Any Python callable distances -> distortions is legal (docs_src/source/mde/index.rst:297-325):
    distances and the scatter still run on the CUDA kernels."""
    pm = _pm()
    rng = np.random.default_rng(9)
    n, p, m = 500, 4000, 3
    e, w, X = _random_problem(n, p, m, rng, push_pull=False)
    wt = torch.tensor(w, device="cuda")

    def f(d):
        return wt * d.pow(2)

    mde = pm.MDE(n, m, torch.tensor(e, device="cuda"), f)
    Xt = torch.tensor(X, device="cuda", requires_grad=True)
    v = mde.average_distortion(Xt)
    v.backward()
    v_ref, g_ref = O.average_distortion(X.astype(np.float64), e, O.FnSpec(O.P_QUADRATIC, w), True)
    np.testing.assert_allclose(v.item(), v_ref, rtol=1e-5)
    np.testing.assert_allclose(Xt.grad.cpu().numpy(), g_ref, atol=2e-5 * float(np.abs(g_ref).max()))


def test_full_size_c2_against_c_oracle():
    """BASELINE config C2 at FULL size (n=70 000, m=2, p~1.55 M, PushAndPull(Log1p, Log)): value and gradient
    of the fused kernel against the C restatement of the reference (oracle/mde_oracle.c, float64)."""
    pm = _pm()
    import bench
    from oracle import c_oracle
    edges, w = bench.c2_edges(0)
    X0 = bench.initial_iterate(0)
    spec = O.FnSpec(O.P_LOG1P, w, (1.5, 0, 0), fn_rep=O.P_LOG, rep=(1.0, 0, 0))
    v_ref, g_ref = c_oracle.average_distortion(X0, edges, spec)
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(bench.N_ITEMS, 2, torch.tensor(edges, device="cuda"), f)
    X = torch.tensor(X0, device="cuda", requires_grad=True)
    v = mde.average_distortion(X)
    v.backward()
    np.testing.assert_allclose(v.item(), v_ref, rtol=1e-5)  # north_star tolerance
    np.testing.assert_allclose(X.grad.cpu().numpy(), g_ref, atol=2e-5 * np.abs(g_ref).max(), rtol=1e-3)
    # bit-exact on edge indices: the caller's int64 list is untouched and per-edge outputs keep its order
    assert torch.equal(mde.edges.cpu(), torch.tensor(edges))
    d = mde.distances(X.detach()).cpu().numpy()
    d_ref = np.linalg.norm(X0[edges[:, 0]].astype(np.float64) - X0[edges[:, 1]].astype(np.float64), axis=1)
    np.testing.assert_allclose(d, d_ref, rtol=1e-5)


@pytest.mark.parametrize("kernel", ["fast", "precise"])
@pytest.mark.parametrize("m", [2, 3])
def test_near_zero_distances_match_reference(golden, m, kernel, monkeypatch):
    """Edges between near-duplicate points (1e-6 <= d <= 1e-1) and exact duplicates (d = 0), attractive and
    repulsive: the MUFU kernels' small-d series for 1 - exp(-d) and the d = 0 mask against the reference's fp64
    run.  The reference's VALUE is -inf when a repulsive edge has d = 0 (log(0)); its gradient is still defined
    (non-finite coefficient -> 1, zero difference vector), so the value is compared on the edges with d > 0."""
    pm = _pm()
    if kernel == "precise":
        monkeypatch.setenv("MDE_B200_KERNEL", "precise")
    g = golden["nearzero"]
    key = "m%d" % m
    edges, X, w = g[key + "/edges"], g[key + "/X"], g[key + "/par0"]
    f = pm.penalties.PushAndPull(torch.tensor(w, device="cuda"), pm.penalties.Log1p, pm.penalties.Log)
    mde = pm.MDE(X.shape[0], m, torch.tensor(edges, device="cuda"), f, pm.Centered())
    Xt = torch.tensor(X, device="cuda", requires_grad=True)
    d = mde.distances(Xt.detach()).cpu().numpy()
    np.testing.assert_allclose(d, g[key + "/f32/distances"], rtol=2e-6, atol=1e-9)
    assert (d == 0).sum() == 2
    # gradient: defined everywhere
    keep = torch.tensor(d > 0, device="cuda")
    sub = pm.MDE(X.shape[0], m, torch.tensor(edges, device="cuda")[keep],
                 pm.penalties.PushAndPull(torch.tensor(w, device="cuda")[keep], pm.penalties.Log1p, pm.penalties.Log),
                 pm.Centered())
    v = sub.average_distortion(Xt) * (int(keep.sum()) / len(edges))  # same divisor as the fixture
    np.testing.assert_allclose(v.item(), float(g[key + "/f64/value_nonzero_edges"]), rtol=1e-5)
    mde.average_distortion(Xt).backward()
    gr = g[key + "/f64/grad"]
    err = np.abs(Xt.grad.cpu().numpy() - gr).max()
    assert err <= 3e-5 * np.abs(gr).max(), (err, np.abs(gr).max())
