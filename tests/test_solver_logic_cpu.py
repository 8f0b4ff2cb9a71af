"""CPU: the scalar solver logic that runs on the device (pymde_b200/csrc/mde_logic.h), exercised
through the library's host-side debug entry points and compared with the oracle's restatement of
pymde/lbfgs.py (strong Wolfe :44-253, two-loop recursion :461-507).  No GPU compute involved."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import mde_oracle as O
from pymde_b200 import _lib
from tests.lbfgs_replay import explicit_two_loop

LS_DONE = 5


def c_strong_wolfe(lib, phi, t0, f0, gtd0, d_norm):
    L = lib.mde_dbg_ls_new(t0, f0, gtd0, d_norm)
    evals = 0
    try:
        while True:
            t = lib.mde_dbg_ls_t(L)
            f, g, fin = phi(t)
            evals += 1
            phase = lib.mde_dbg_ls_step(L, float(f), float(g), int(fin))
            if phase == LS_DONE:
                break
            assert evals < 400
        ta, fa, fe, err = C.c_double(), C.c_double(), C.c_int(), C.c_int()
        lib.mde_dbg_ls_result(L, C.byref(ta), C.byref(fa), C.byref(fe), C.byref(err))
        return ta.value, fa.value, evals, err.value
    finally:
        lib.mde_dbg_ls_free(L)


def make_phi(kind, rng):
    a = rng.uniform(0.2, 5.0)
    b = rng.uniform(0.5, 3.0)
    if kind == "quad":
        f = lambda t: (b * (t - a) ** 2, 2 * b * (t - a))
    elif kind == "quartic":
        f = lambda t: ((t - a) ** 4 + 0.3 * math.sin(3 * t), 4 * (t - a) ** 3 + 0.9 * math.cos(3 * t))
    elif kind == "abs":
        f = lambda t: (b * abs(t - a) + 0.1 * t * t, b * np.sign(t - a) + 0.2 * t)
    elif kind == "barrier":  # NaN beyond t >= a (outside the domain), like a log barrier
        c = 1.0 / a + b
        f = lambda t: ((-math.log(a - t) - c * t, 1.0 / (a - t) - c) if t < a else (float("nan"), float("nan")))
    elif kind == "steep":
        f = lambda t: (math.exp(-b * t) + 0.05 * t, -b * math.exp(-b * t) + 0.05)
    else:
        raise ValueError(kind)

    def phi(t):
        v, g = f(float(t))
        v = float(np.float32(v))  # losses are fp32 in the reference
        g = np.float32(g)
        return v, g, bool(np.isfinite(g))
    return phi


@pytest.mark.parametrize("seed", [0, 1000])
@pytest.mark.parametrize("kind", ["quad", "quartic", "abs", "barrier", "steep"])
def test_strong_wolfe_state_machine_matches_oracle(kind, seed):
    lib = _lib.load()
    rng = np.random.default_rng({"quad": 11, "quartic": 23, "abs": 37, "barrier": 41, "steep": 53}[kind] + seed)
    checked = 0
    for _ in range(60):
        phi = make_phi(kind, rng)
        f0, g0, _ = phi(0.0)
        if not (g0 < 0) or not np.isfinite(f0):
            continue
        t0 = float(rng.choice([1.0, 0.05, 7.0, 1e-3]))
        d_norm = np.float32(rng.uniform(0.1, 10))
        try:
            f_ref, t_ref, _ = O.strong_wolfe(phi, t0, f0, g0, d_norm, sdt=np.float32)
            err_ref = 0
        except O.SolverError:
            err_ref = 1
        t_c, f_c, evals, err_c = c_strong_wolfe(lib, phi, t0, f0, float(g0), float(d_norm))
        assert err_c == err_ref
        if not err_ref:
            assert t_c == pytest.approx(float(t_ref), rel=2e-5, abs=1e-12), (kind, t0)
            # the accepted value is phi at the accepted step (the barrier is steep near its pole, so compare
            # the values through the steps: equal steps to 2e-5 => values within the local slope times that)
            assert f_c == pytest.approx(phi(t_c)[0], rel=1e-6, abs=1e-9)
            slope = abs(float(phi(t_c)[1]))
            assert abs(f_c - float(f_ref)) <= 1e-4 * abs(float(f_ref)) + 1e-7 + 4e-5 * slope * abs(t_c)
        checked += 1
    assert checked > 20


@pytest.mark.parametrize("memory", [1, 3, 10])
def test_gram_form_two_loop_matches_explicit(memory):
    """Drive the device-side history logic with a synthetic gradient sequence; the direction
    rebuilt from its coefficients must equal the explicit two-loop recursion on the same pairs,
    including eviction when the memory is full and rejection of pairs with y.s <= 1e-10."""
    lib = _lib.load()
    rng = np.random.default_rng(memory)
    N, MAXM = 40, 33
    A = rng.standard_normal((N, N))
    A = A @ A.T / N + np.eye(N)  # SPD quadratic: g = A x
    B = lib.mde_dbg_lbfgs_new(memory)
    Sphys = np.zeros((memory + 1, N))
    Yphys = np.zeros((memory + 1, N))
    pairs = []  # explicit history (oldest..newest)
    H_diag = 1.0
    x = rng.standard_normal(N)
    g = A @ x
    arr = lambda: (C.c_double * MAXM)()
    d_prev = t_prev = g_prev = None
    try:
        for it in range(25):
            sj_yc, yj_yc, sc_yj, sj_g, yj_g = arr(), arr(), arr(), arr(), arr()
            ys = yy = sc_g = yc_g = 0.0
            if it > 0:
                y = g - g_prev
                s = t_prev * d_prev
                if it == 7:  # force a rejected pair (y.s <= 1e-10)
                    y = -y
                cand = lib.mde_dbg_lbfgs_cand(B)
                Sphys[cand], Yphys[cand] = s, y
                ys, yy, sc_g, yc_g = float(y @ s), float(y @ y), float(s @ g), float(y @ g)
                for j, q in enumerate(order_now):
                    sj_yc[j] = float(Sphys[q] @ y)
                    yj_yc[j] = float(Yphys[q] @ y)
                    sc_yj[j] = float(s @ Yphys[q])
                    sj_g[j] = float(Sphys[q] @ g)
                    yj_g[j] = float(Yphys[q] @ g)
                if ys > 1e-10:
                    if len(pairs) == memory:
                        pairs.pop(0)
                    pairs.append((s.copy(), y.copy()))
                    H_diag = float(np.float32(ys) / np.float32(yy))
            count, cand_o, cg = C.c_int(), C.c_int(), C.c_double()
            order = (C.c_int * MAXM)()
            cs, cy = arr(), arr()
            lib.mde_dbg_lbfgs_step(B, ys, yy, sc_g, yc_g, sj_yc, yj_yc, sc_yj, sj_g, yj_g,
                                   C.byref(count), C.byref(cand_o), order, C.byref(cg), cs, cy)
            order_now = [order[j] for j in range(count.value)]
            assert count.value == len(pairs)
            d = cg.value * g
            for j, q in enumerate(order_now):
                d = d + cs[j] * Sphys[q] + cy[j] * Yphys[q]
            d_ref = explicit_two_loop(g, [p[0] for p in pairs], [p[1] for p in pairs], H_diag) if pairs else -g
            np.testing.assert_allclose(d, d_ref, rtol=1e-8, atol=1e-10)
            # take a step
            t_prev = 0.7 if it else min(1.0, 1.0 / np.abs(g).sum())
            d_prev, g_prev = d, g
            x = x + t_prev * d
            g = A @ x
    finally:
        lib.mde_dbg_lbfgs_free(B)


def test_library_exports_every_declared_symbol():
    """include/mde_b200.h <-> libmde_b200.so: every declared entry point resolves."""
    import re, os
    lib = _lib.load()
    hdr = open(os.path.join(os.path.dirname(_lib._HERE), "include", "mde_b200.h")).read()
    names = set(re.findall(r"\b(mde_[a-z_0-9]+)\s*\(", hdr)) - {"mde_allreduce_fn"}
    assert names, "no declarations found"
    for n in sorted(names):
        assert hasattr(lib, n), n
        assert n in _lib.SIGNATURES, "binding missing for " + n
    assert lib.mde_abi_version() == 1
    assert lib.mde_error_string(-3).decode().startswith("mde:")
