"""The fp64 oracle (oracle/mde_oracle.py::eval_function) against the reference on the function matrix.

tests/golden/function_matrix.npz holds the unmodified reference's f and autograd f' in fp32 and fp64 for every
table function at every exponent branch, threshold, alpha, gamma, weight sign and distance regime of
tests/function_matrix_cases.py.  The GPU tests judge the kernels by these columns and by the oracle, so the oracle
must first agree with the reference at every point:

  * non-finite values: the same class (+inf, -inf or NaN) in fp32 and in fp64;
  * finite values, r64 = the reference in fp64, r32 = the reference in fp32, o = the oracle in precision dt:

        |o - r64| <= c |r32 - r64| + 16 ulp_dt(r64) + 16 eps_dt max(1, |par0|)

    c = 2 in fp32: the fp32 oracle is at most twice as far from the fp64 reference as the fp32 reference itself.
    c = 2^-27 in fp64: the fp64 reference runs the same operations as its fp32 run, so where they cancel (torch's
    chain rule for LogRatio, the logsumexp of SoftFractional) its error is its fp32 error scaled by eps64 / eps32 =
    2^-29, and the closed forms of the oracle do not cancel; 4x headroom.
    The last term is the absolute rounding of the terms a value is summed from (weights and deviations are O(1)):
    the reference rounds log(1 + e^z) to exactly 0 for z < -37 (logsumexp) and e^-x (1 - e^-x)^-1 to exactly 0 when
    1 - e^-x rounds to 1 (expm1's derivative), where the true value is tiny but not 0.
"""
import os

import numpy as np
import pytest

from oracle import mde_oracle as O
from tests import function_matrix_cases as FM

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "function_matrix.npz"))


def spec_of(name):
    fn = GOLD[name + "/fn"]
    par1 = GOLD[name + "/par1"] if name + "/par1" in GOLD.files else None
    if fn[2]:
        return O.FnSpec(fn[0], GOLD[name + "/par0"], GOLD[name + "/att"], fn_rep=fn[1], rep=GOLD[name + "/rep"])
    return O.FnSpec(fn[0], GOLD[name + "/par0"], GOLD[name + "/att"], par1=par1)


def nonfinite_class(x):
    """0 finite, 1 +inf, 2 -inf, 3 NaN"""
    x = np.asarray(x)
    return np.where(np.isnan(x), 3, np.where(np.isposinf(x), 1, np.where(np.isneginf(x), 2, 0)))


def bound(name, col, dtype):
    """the finite-value bound of the module docstring, per point"""
    r64 = GOLD["%s/f64/%s" % (name, col)].astype(np.float64)
    r32 = GOLD["%s/f32/%s" % (name, col)].astype(np.float64)
    with np.errstate(invalid="ignore"):
        e32 = np.where(np.isfinite(r32) & np.isfinite(r64), np.abs(r32 - r64), 0.0)
    c = 2.0 if dtype is np.float32 else 2.0 ** -27
    ulp = np.spacing(np.abs(np.where(np.isfinite(r64), r64, 0.0)).astype(dtype)).astype(np.float64)
    eps = float(np.finfo(dtype).eps)
    return c * e32 + 16 * ulp + 16 * eps * np.maximum(1.0, np.abs(GOLD[name + "/par0"].astype(np.float64)))


def test_fixture_covers_the_matrix():
    names = {c.name for c in FM.CASES}
    assert names == {k.split("/")[0] for k in GOLD.files}
    for c in FM.CASES:
        d, par0, _ = FM.points(c)
        np.testing.assert_array_equal(GOLD[c.name + "/d"], d)
        np.testing.assert_array_equal(GOLD[c.name + "/par0"].view(np.uint32), par0.view(np.uint32))  # -0.0 kept
    # every pow_pair branch and powf, for every function that takes an exponent
    for fam in ("pen_power", "pen_log1p", "pen_log", "pen_invpower", "pen_logratio", "loss_power"):
        assert {"%s_%g" % (fam, e) for e in FM.EXPONENTS} <= names
    assert any(np.any((GOLD[n + "/d"] == 0)) for n in names)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", [c.name for c in FM.CASES])
def test_oracle_matches_reference(name, dtype):
    tag = "f64" if dtype is np.float64 else "f32"
    d = GOLD[name + "/d"]
    with np.errstate(all="ignore"):
        out = O.eval_function(spec_of(name), d, dtype)
    for col, o in zip(("f", "fp"), out):
        r = GOLD["%s/%s/%s" % (name, tag, col)]
        assert o.dtype == dtype
        cls_o, cls_r = nonfinite_class(o), nonfinite_class(r)
        bad = np.flatnonzero(cls_o != cls_r)
        assert not len(bad), (col, [(float(d[i]), o[i], r[i]) for i in bad[:5]])
        fin = cls_r == 0
        r64 = GOLD["%s/f64/%s" % (name, col)].astype(np.float64)
        fin &= np.isfinite(r64)
        err = np.abs(o.astype(np.float64) - r64)
        tol = bound(name, col, dtype)
        bad = np.flatnonzero(fin & ~(err <= tol))
        assert not len(bad), (col, [(float(d[i]), float(o[i]), float(r64[i]), float(tol[i])) for i in bad[:5]])
