"""Generate tests/golden/function_matrix.npz by RUNNING THE UNMODIFIED REFERENCE (cvxgrp/pymde v0.2.1) on the
function matrix of tests/function_matrix_cases.py.

    PYMDE_REFERENCE=<reference checkout> python tests/golden/make_function_matrix_golden.py

For every case it evaluates the reference's `penalties` / `losses` module in fp32 and in fp64 on the same fp32
distances and parameters, the way make_golden.py does, and records f and the autograd derivative f' = df/dd.  Per
case `<name>/...`:
  d, par0                 the points (fp32)
  par1                    WeightedQuadratic only: the weights the fp64 function holds (given, or 1 / delta^2)
  fn                      int32 [fn_att, fn_rep, push_pull] (ids of include/mde_b200.h)
  att, rep                float64 [3]: the scalar parameters as the reference holds them
  f32/f, f32/fp           the reference in fp32
  f64/f, f64/fp           the reference in fp64 (the exact arbiter)
The script is deterministic: two runs write identical arrays.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
from oracle.ref_loader import load_reference  # noqa: E402
from oracle import mde_oracle as O  # noqa: E402
from tests import function_matrix_cases as FM  # noqa: E402

pymde = load_reference()
assert pymde is not None, "reference not importable"
torch.set_num_threads(1)


def run(case, d, par0, par1, dtype):
    p0 = torch.tensor(par0, dtype=dtype)
    p1 = None if par1 is None else torch.tensor(par1, dtype=dtype)
    f = FM.build(pymde, case, p0, p1)
    dd = torch.tensor(d, dtype=dtype).requires_grad_(True)
    val = f(dd)
    val.sum().backward()
    return f, val.detach().numpy(), dd.grad.numpy()


def main():
    out = {}
    for case in FM.CASES:
        d, par0, par1 = FM.points(case)
        key = case.name
        out[key + "/d"], out[key + "/par0"] = d, par0
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            f, val, fp = run(case, d, par0, par1, dtype)
            out["%s/%s/f" % (key, tag)], out["%s/%s/fp" % (key, tag)] = val, fp
            spec = O.spec_from_function(f)
            if tag == "f32":
                out[key + "/fn"] = np.array([spec.fn_att, spec.fn_rep, int(spec.push_pull)], np.int32)
                out[key + "/att"] = np.array(spec.att, np.float64)
                out[key + "/rep"] = np.array(spec.rep, np.float64)
            elif spec.par1 is not None:  # the second weight array the function holds (given, or 1 / delta^2)
                out[key + "/par1"] = np.asarray(spec.par1, np.float64)
    np.savez_compressed(os.path.join(HERE, "function_matrix.npz"), **out)
    print("function_matrix.npz: %d cases, %d points" % (
        len(FM.CASES), sum(len(out[c.name + "/d"]) for c in FM.CASES)))


if __name__ == "__main__":
    main()
