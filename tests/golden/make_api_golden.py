"""Record the public surface of the UNMODIFIED REFERENCE (cvxgrp/pymde v0.2.1) for tests/test_api_surface_cpu.py.

    PYMDE_REFERENCE=<reference checkout with its Cython extension built> python tests/golden/make_api_golden.py

Outputs (committed): tests/golden/api_surface.json (parameter lists and public names) and api_helpers.npz (inputs and
reference outputs of the host-side helpers).  The tests read only these files.
"""
import inspect
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
from oracle.ref_loader import load_reference  # noqa: E402
import pymde_b200 as pm  # noqa: E402

ref = load_reference()
assert ref is not None, "reference not importable"

OUT_OF_SCOPE = {"latexify", "plot", "datasets", "experiment_utils"}  # plotting / downloads (SURVEY section 2)
PENALTIES = ("Linear", "Quadratic", "Cubic", "Power", "Huber", "Logistic", "Sigmoid", "Hinge", "Log1p", "Log",
             "InvPower", "LogRatio", "PushAndPull")
LOSSES = ("Absolute", "Quadratic", "WeightedQuadratic", "Huber", "Cubic", "Power", "Logistic", "Fractional",
          "SoftFractional")
MODULES = ("penalties", "losses", "constraints", "preprocess", "recipes", "quadratic")


def params(f):
    return [p for p in inspect.signature(f).parameters if p != "self"]


def signatures():
    fns = {
        "MDE.__init__": ref.MDE.__init__, "MDE.embed": ref.MDE.embed,
        "MDE.average_distortion": ref.MDE.average_distortion, "MDE.distortions": ref.MDE.distortions,
        "MDE.distances": ref.MDE.distances, "MDE.differences": ref.MDE.differences,
        "MDE.high_distortion_pairs": ref.MDE.high_distortion_pairs, "preserve_neighbors": ref.preserve_neighbors,
        "preserve_distances": ref.preserve_distances, "laplacian_embedding": ref.laplacian_embedding,
        "Anchored": ref.Anchored.__init__, "Graph.from_edges": ref.Graph.from_edges,
        "quadratic.spectral": ref.quadratic.spectral, "pca": ref.pca, "align": ref.align, "rotate": ref.rotate,
        "util.proj_standardized": ref.util.proj_standardized,
        "preprocess.dissimilar_edges": ref.preprocess.dissimilar_edges,
        "preprocess.graph.shortest_paths": ref.preprocess.graph.shortest_paths, "Graph.draw": ref.Graph.draw,
    }
    for cls in PENALTIES:
        fns["penalties." + cls] = getattr(ref.penalties, cls).__init__
    for cls in LOSSES:
        fns["losses." + cls] = getattr(ref.losses, cls).__init__
    for name in ("sample_edges", "k_nearest_neighbors", "distances"):
        fns["preprocess." + name] = getattr(ref.preprocess, name)
    return {k: params(f) for k, f in fns.items()}


def public_names():
    top = sorted(name for name in dir(ref) if not name.startswith("_") and name not in OUT_OF_SCOPE and
                 (inspect.isfunction(getattr(ref, name)) or inspect.isclass(getattr(ref, name))))
    mods = {}
    for mod in MODULES:
        r = getattr(ref, mod)
        mods[mod] = sorted(
            name for name in dir(r) if not name.startswith("_") and
            (inspect.isfunction(getattr(r, name)) or inspect.isclass(getattr(r, name))) and
            getattr(getattr(r, name), "__module__", "").startswith("pymde"))
    return {"top_level": top, "modules": mods}


def helpers():
    out = {}
    torch.manual_seed(0)
    w, d = torch.randn(64), torch.rand(64) * 3
    out["w"], out["d"] = w.numpy(), d.numpy()
    for i, (name, args) in enumerate((("Sigmoid", (1.0, 2.0)), ("Sigmoid", (0.5,)), ("Hinge", (1.0,)),
                                      ("Hinge", (1.5, 0.2)))):
        out["penalty%d" % i] = getattr(ref.penalties, name)(w, *args)(d).numpy()
    X2, X3 = torch.randn(9, 2), torch.randn(9, 3)
    deg = torch.tensor([10.0, 20.0, 30.0])
    out["X2"], out["X3"], out["deg"] = X2.numpy(), X3.numpy(), deg.numpy()
    out["rotate2"] = ref.rotate(X2, torch.tensor(33.0)).numpy()
    out["rotate3"] = ref.rotate(X3, deg).numpy()
    out["random_edges"] = ref.util.random_edges(50, 100, seed=3).numpy()
    e, wt = torch.tensor([[0, 1], [1, 3]]), torch.tensor([1.0, 2.0])
    out["adjacency"] = ref.util.adjacency_matrix(5, 2, e, wt).toarray()
    Xq = torch.tensor([[1.0, 1.0], [1.0, -1.0], [-1.0, 1.0], [-1.0, -1.0]])
    out["Xq_in_stdemb"] = np.array(bool(ref.util.in_stdemb(Xq)))
    for seed in range(4):
        torch.manual_seed(seed)
        Xs = ref.util.proj_standardized(torch.randn(40, 2), demean=True)
        out["Xs%d" % seed] = Xs.numpy()
        out["Xs%d_in_stdemb" % seed] = np.array(bool(ref.util.in_stdemb(Xs)))
    Y = torch.randn(30, 6)
    a = ref.pca(Y, 2)
    b = pm.pca(Y, 2)  # the target of the alignment below: any 30 x 2 matrix serves
    out["Y"], out["pca"], out["align_target"] = Y.numpy(), a.numpy(), b.numpy()
    out["align"] = ref.align(a, b).numpy()
    return out


if __name__ == "__main__":
    with open(os.path.join(HERE, "api_surface.json"), "w") as fh:
        json.dump({"signatures": signatures(), "names": public_names()}, fh, indent=1, sort_keys=True)
        fh.write("\n")
    np.savez_compressed(os.path.join(HERE, "api_helpers.npz"), **helpers())
    print("wrote api_surface.json, api_helpers.npz")
