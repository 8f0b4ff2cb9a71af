"""Why the sparse exact k-nearest-neighbour searches certify every row, on the CPU; and the ABI of their `_ex` entries.

The tile kernels of csrc/mde_knn_sparse.cu rank candidate x of query q by s(x) = fl(||x||^2~ - 2 <q, x>~): ||x||^2~ is
the fp64 sum of squares rounded once to fp32, <., .>~ the cross term of the bf16 hi / lo split (x = h + l + r,
|r| <= 2^-16 |x|; products h h + h l + l h, exact in fp32, accumulated in fp32), and the score is one fma.  They keep
the KK best scores per row (32, 96 or 288) and re-rank those by the exact distance.  The columns are not centred (that
would densify the matrix), so a column shared by every row far from the origin -- a year, a latitude, a constant bias
feature -- makes ||x||^2 large against the neighbour distances, and the kept list is rounding noise.  The simulation
below keeps 32 and reproduces the table of the families at k = 15.

The certificate needs a bound E(q) >= |s(x) - S(x)|, S(x) = ||x||^2 - 2 <q, x> the exact score, for every x that can
enter the list.  With u = 2^-24 and m = 3 nnz(q), for every x with ||x|| <= R:

  split        the dropped l_q l_x and the residuals: per element at most (2^-16 (1 + 2^-8)^2 + 2 2^-16 (1 + 2^-8))
               |q_j||x_j| < 3.1 2^-16 |q_j||x_j|; by Cauchy-Schwarz the sum is at most 3.1 2^-16 |q||x|.
  accumulation the fp32 sum of the products adds at most 2 u per addition (2 u allows for tensor cores that truncate
               rather than round).  A product with an element q_j = 0 is an exact zero (h = l = 0), and adding an exact
               zero is exact, so only m = 3 nnz(q) addends count, not 3 d: at most 2 u m sum |products| <= 2 u m |q||x|
               to first order.  A bound in d would certify nothing at d = 10^5.
  norm         the fp64 sum of at most d squares (relative (d + 6) 2^-53) rounded once to fp32 (u).
  score        the fma: at most u (||x||^2 + 2 |q||x|).
  subnormals   a split part below 2^-126, flushed or not, errs by at most 2^-126 per element: eta = 2^-126 sqrt(nnz(q))
               per unit of |q| + |x|; underflowing products at most 2^-126 each, norms 2^-149.

So E(q) = sigma (2 (a_cross |q| R + eta (|q| + R)) + a_norm R^2 + a_abs) with a_cross = 3.1 2^-16 + 2 u m + u,
a_norm = 2 u + (d + 6) 2^-53, a_abs = 2 m 2^-126 + 2 2^-149, and sigma = 2 for the second-order factors.

Which R: a row x can enter the list only if its fp32 distance is at most d2_k, the k-th re-ranked one, and then
||x|| <= ||q|| + ||q - x|| <= R = sqrt(qn / (1 - a_norm)) + sqrt(d2_k / (1 - delta)) (qn the fp32 norm of q; the kernel
adds 2^-149 to both and a relative 2^-40).  The global maximum norm would let a few long documents decertify every
row; R depends on the row alone.

A row is certified when (d2_k + 2^-149) (1 + delta) / (1 - delta) - qn + E < t - E and R^2 < 2^125, t the worst
(KK-th) kept score and delta = u + (d + 2) 2^-53 the re-rank's relative rounding: a row not kept with ||x|| <= R scored
at least t, so its exact distance is at least t - E + qn - E, more than d2_k by the margin, and a row with ||x|| > R
is farther than d2_k anyway.  The check below measures the simulated score error on every row and on every candidate
within R of every family against E / sigma: the bound holds without the safety factor.  It also predicts the share of
rows certified: all of them on the ordinary continuous families."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from pymde_b200 import _lib
from tests.test_gpu_knn_csr_offset import FAR, ORDINARY, TIE_HEAVY, family

U = 2.0 ** -24
SIGMA = 2.0
N_SIM = 1500


def split(X):
    h = X.to(torch.bfloat16).float()
    return h, (X - h).to(torch.bfloat16).float()


def simulate(A):
    """(fp32 dense X, tile scores s [n, n] fp32 with +inf on the diagonal, fp32 norms, fp64 exact scores S)."""
    X = torch.from_numpy(A.toarray().astype(np.float32))
    Xd = X.double()
    norms = (Xd * Xd).sum(1).float()
    h, l = split(X)
    cross = h @ h.T + h @ l.T + l @ h.T  # fp32 products and sums
    s = torch.addcmul(norms[None, :], cross, torch.tensor(-2.0))  # one rounding, as the tile's fma
    s.fill_diagonal_(float("inf"))
    S = (Xd * Xd).sum(1)[None, :] - 2.0 * Xd @ Xd.T
    return X, s, norms, S


def exact_d2(X):
    Xd = X.double()
    D = ((Xd[:, None, :] - Xd[None, :, :]) ** 2).sum(-1) if X.shape[1] <= 64 else (
        (Xd * Xd).sum(1)[:, None] + (Xd * Xd).sum(1)[None, :] - 2.0 * Xd @ Xd.T).clamp(min=0.0)
    D.fill_diagonal_(float("inf"))
    return D


def exact_rows(X, rows, cols):
    """fp64 sum (x_r - x_c)^2 of rows [r] against cols [r, m] (no cancellation: the search's own distances)."""
    Xd = X.double()
    return ((Xd[rows][:, None, :] - Xd[cols]) ** 2).sum(-1)


def kept_and_reranked(X, s, k, kk=32):
    """The kept list (top kk by (score, index)), its worst score t and the re-rank's k-th fp32 distance."""
    n = X.shape[0]
    order = torch.from_numpy(np.lexsort((np.broadcast_to(np.arange(n), (n, n)), s.numpy()), axis=1)[:, :kk].copy())
    t = torch.gather(s, 1, order).max(1)[0].double()
    d2 = exact_rows(X, torch.arange(n), order).float()
    d2k = torch.sort(d2, 1)[0][:, k - 1].double()
    return order, t, d2k


def wrong_fraction(A, k=15):
    """Fraction of rows whose k-th re-ranked distance (top 32 by the simulated score) is farther than the true."""
    X, s, _, _ = simulate(A)
    _, _, got = kept_and_reranked(X, s, k)
    D = exact_d2(X)
    want = torch.topk(D, k, dim=1, largest=False)[0][:, k - 1]
    return float((got > want * (1 + 1e-6) + 1e-30).double().mean())


def bound(nnz, d, qn, d2k):
    """(E, R, delta) of knn_csr_certify_kernel, sigma included; nnz, qn, d2k are per-row tensors."""
    tiny = 2.0 ** -149
    m = 3.0 * nnz
    a_cross = 3.1 * 2.0 ** -16 + 2 * U * m + U
    eta = 2.0 ** -126 * torch.sqrt(m / 3.0)
    a_norm = 2 * U + (d + 6.0) * 2.0 ** -53
    a_abs = 2 * m * 2.0 ** -126 + 2 * tiny
    delta = U + (d + 2.0) * 2.0 ** -53
    qa = torch.sqrt((qn + tiny) / (1 - a_norm)) * (1 + 2.0 ** -40)
    R = qa + torch.sqrt((d2k + tiny) / (1 - delta)) * (1 + 2.0 ** -40)
    E = SIGMA * (2 * (a_cross * qa * R + eta * (qa + R)) + a_norm * R * R + a_abs)
    return E, R, delta


def certified(A, k=15, kk=32):
    X, s, norms, _ = simulate(A)
    _, t, d2k = kept_and_reranked(X, s, k, kk)
    nnz = torch.from_numpy(np.diff(A.indptr).astype(np.float64))
    qn = norms.double()
    E, R, delta = bound(nnz, A.shape[1], qn, d2k)
    lhs = (d2k + 2.0 ** -149) * (1 + delta) / (1 - delta) - qn + E
    return (lhs < t - E) & (R * R < 2.0 ** 125)


# the failure table (n = 1 500, k = 15: share of rows whose 15 neighbours are wrong)
@pytest.mark.parametrize("name,low,high", [("latlong_onehot", 0.9, 1.0), ("year_counts", 0.5, 1.0),
                                           ("count_docs", 0.0, 0.0), ("uniform", 0.0, 0.0)])
def test_failure_table(name, low, high):
    frac = wrong_fraction(family(name, n=N_SIM))
    print(name, "rows with wrong neighbours:", frac)
    assert low <= frac <= high, frac


@pytest.mark.parametrize("name", FAR + ORDINARY + TIE_HEAVY + ["huge_rows"])
def test_score_error_is_within_the_certificate_bound(name):
    A = family(name, n=N_SIM)
    X, s, norms, S = simulate(A)
    n, d = A.shape
    nnz = torch.from_numpy(np.diff(A.indptr).astype(np.float64))
    D = exact_d2(X)
    d2k = torch.topk(D, 15, dim=1, largest=False)[0][:, 14].float().double()  # the k-th fp32 distance
    qn = norms.double()
    E, R, _ = bound(nnz, d, qn, d2k)
    E = E / SIGMA  # without the safety factor
    xn = (X.double() ** 2).sum(1).sqrt()
    within = (xn[None, :] <= R[:, None]) & ~torch.eye(n, dtype=torch.bool)
    ok_rows = torch.isfinite(E)
    within &= ok_rows[:, None]
    err = (s.double() - S).abs()
    assert bool(torch.isfinite(err[within]).all())
    worst = float((err / E[:, None])[within].max()) if bool(within.any()) else 0.0
    print(name, "largest error / bound:", worst)
    assert worst <= 1.0, worst
    # the fp32 norms of the queries too (the certificate's right-hand E)
    q = ok_rows
    assert bool(((qn - (X.double() ** 2).sum(1)).abs()[q] <= E[q]).all())
    if name == "huge_rows":  # only the rows whose norm overflows fp32 have no finite bound
        assert int((~torch.isfinite(E)).sum()) == int((~torch.isfinite(norms)).sum()) > 0


@pytest.mark.parametrize("name", ORDINARY)
def test_ordinary_families_certify(name):
    """The bound in nnz(q), not d, over the rows within R: every row of the ordinary continuous families certifies."""
    ok = certified(family(name, n=N_SIM))
    print(name, "rows certified:", float(ok.double().mean()))
    assert float(ok.double().mean()) >= 0.99


@pytest.mark.parametrize("name", FAR)
def test_far_families_fail_the_certificate(name):
    ok = certified(family(name, n=N_SIM))
    print(name, "rows certified:", float(ok.double().mean()))
    assert float(ok.double().mean()) < 0.5


def test_a_bound_in_d_would_certify_nothing_at_large_d():
    """Rows of 2 000 N(0, 1) values among 10^5 features (2 % dense) lie about 4 000 apart in squared distance, with a
    standard deviation of about 89 (sqrt(2 * 4 000)).  The certificate needs the gap between the k-th and the KK-th
    neighbour to exceed about 4 E.  With m = 3 nnz(q) that is 57, within one standard deviation; with m = 3 d it would
    be 2 700, more than the whole spread of the distances (6 standard deviations), and no row would certify."""
    one = torch.ones(1)
    E_nnz, _, _ = bound(2000 * one, 10 ** 5, 2000 * one, 3600 * one)
    E_d, _, _ = bound(10 ** 5 * one, 10 ** 5, 2000 * one, 3600 * one)
    sd = (2 * 4000) ** 0.5
    assert float(4 * E_nnz) < sd and float(4 * E_d) > 6 * sd, (float(E_nnz), float(E_d))


# --- ABI: the _ex entries --------------------------------------------------------------------------------------------

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # non-null, 1024-byte aligned: never dereferenced, every check below fails before a CUDA call
FULL = {"mde_knn_csr_ex": 24, "mde_knn_csr_wide_ex": 64, "mde_knn_csr_long_ex": 256}


def test_ex_entries_are_exported_and_the_abi_version_is_unchanged():
    lib = _lib.load()
    assert lib.mde_abi_version() == 1
    with open(os.path.join(REPO, "include", "mde_b200.h")) as fh:
        header = fh.read()
    for name in list(FULL) + ["mde_knn_csr_rows_ex"]:
        assert name in _lib.SIGNATURES and getattr(lib, name) is not None
        assert "int %s(" % name in header


def _outputs():
    return np.full(64 * 8, -7, np.int32), np.full(64 * 8, -7.0, np.float32), C.c_int(-5)


@pytest.mark.parametrize("name", sorted(FULL))
def test_full_ex_entries_refuse_bad_arguments_before_any_cuda_call(name):
    lib = _lib.load()
    fn = getattr(lib, name)
    max_k = FULL[name]
    n, d, nnz = 1000, 30, 500
    oi, od, fb = _outputs()

    def call(n=n, d=d, nnz=nnz, k=5, indptr=FAKE, indices=FAKE, values=FAKE, out_i=oi.ctypes.data,
             out_d=od.ctypes.data, ws=FAKE, ws_bytes=1 << 40):
        return fn(indptr, indices, values, n, d, nnz, k, out_i, out_d, ws, ws_bytes, None, C.byref(fb))

    for kw in [dict(k=0), dict(k=max_k + 1), dict(n=1, k=1), dict(n=10, k=10), dict(d=0), dict(nnz=-1),
               dict(indptr=None), dict(indices=None), dict(values=None), dict(out_i=None), dict(out_d=None),
               dict(ws=None)]:
        assert call(**kw) == _lib.MDE_E_INVALID, kw
    assert (oi == -7).all() and (od == -7.0).all() and fb.value == -5  # nothing written


def test_rows_ex_refuses_bad_arguments_before_any_cuda_call():
    lib = _lib.load()
    n, d, nnz = 1000, 30, 500
    oi, od, fb = _outputs()

    def call(rb=0, re=10, k=5, n=n, ws=FAKE, ws_bytes=1 << 40, indptr=FAKE):
        return lib.mde_knn_csr_rows_ex(indptr, FAKE, FAKE, n, d, nnz, rb, re, k, oi.ctypes.data, od.ctypes.data, ws,
                                       ws_bytes, None, C.byref(fb))

    for kw in [dict(rb=-1), dict(rb=5, re=5), dict(re=n + 1), dict(k=0), dict(k=257), dict(n=10, re=10, k=10),
               dict(ws=None), dict(indptr=None), dict(ws_bytes=0), dict(ws=FAKE + 8)]:
        assert call(**kw) == _lib.MDE_E_INVALID, kw
    assert (oi == -7).all() and (od == -7.0).all() and fb.value == -5


@pytest.mark.parametrize("k", [5, 40, 100])
def test_full_workspace_grows_by_the_certificate_and_monotonically(k):
    """The full searches' workspace: the certificate adds a header and one row id per row; it grows with n."""
    lib = _lib.load()
    name = "mde_knn_csr%s_ws_bytes" % ("_long" if k > 64 else "_wide" if k > 24 else "")
    if lib.mde_knn_csr_ws_bytes(1000, 30, 500, None) != _lib.MDE_E_INVALID:
        pytest.fail("a null size pointer must be refused")
    sizes = []
    for n in (k + 1, 1000, 20000, 100000, 100001, 500000):
        need = C.c_size_t(0)
        rc = getattr(lib, name)(n, 30000, n * 40, C.byref(need))
        if rc != 0:  # the sort-scratch query needs a device on a machine without one
            pytest.skip("workspace query needs a CUDA device here")
        sizes.append(need.value)
    assert all(b >= a for a, b in zip(sizes, sizes[1:])), sizes
