"""CPU: the package is a drop-in for the reference's public surface.  Signatures and public names are compared with
those of the unmodified reference, and the host-side helpers that do not need the GPU are checked against it value
for value.  What the reference gives is stored in tests/golden/api_surface.json and api_helpers.npz
(tests/golden/make_api_golden.py)."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

import pymde_b200 as pm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ref():
    with open(os.path.join(GOLDEN, "api_surface.json")) as fh:
        return json.load(fh)


@pytest.fixture(scope="module")
def helpers():
    return dict(np.load(os.path.join(GOLDEN, "api_helpers.npz")))


def _params(f):
    return [p for p in inspect.signature(f).parameters if p != "self"]


def test_public_signatures_match_the_reference(ref):
    sig = ref["signatures"]
    ours = {
        "MDE.__init__": pm.MDE.__init__, "MDE.embed": pm.MDE.embed, "MDE.average_distortion": pm.MDE.average_distortion,
        "MDE.distortions": pm.MDE.distortions, "MDE.distances": pm.MDE.distances, "MDE.differences": pm.MDE.differences,
        "MDE.high_distortion_pairs": pm.MDE.high_distortion_pairs, "preserve_neighbors": pm.preserve_neighbors,
        "preserve_distances": pm.preserve_distances, "laplacian_embedding": pm.laplacian_embedding,
        "Anchored": pm.Anchored.__init__, "Graph.from_edges": pm.Graph.from_edges,
        "quadratic.spectral": pm.quadratic.spectral, "pca": pm.pca, "align": pm.align, "rotate": pm.rotate,
        "util.proj_standardized": pm.util.proj_standardized,
        "preprocess.dissimilar_edges": pm.preprocess.dissimilar_edges,
    }
    for cls in ("Linear", "Quadratic", "Cubic", "Power", "Huber", "Logistic", "Sigmoid", "Hinge", "Log1p", "Log",
                "InvPower", "LogRatio", "PushAndPull"):
        ours["penalties." + cls] = getattr(pm.penalties, cls).__init__
    for cls in ("Absolute", "Quadratic", "WeightedQuadratic", "Huber", "Cubic", "Power", "Logistic", "Fractional",
                "SoftFractional"):
        ours["losses." + cls] = getattr(pm.losses, cls).__init__
    for name, f in ours.items():
        assert sig[name] == _params(f), name
    # same leading parameters; ours may add a trailing `device=` (the data always ends up on a CUDA device)
    for name in ("sample_edges", "k_nearest_neighbors", "distances"):
        a, b = sig["preprocess." + name], _params(getattr(pm.preprocess, name))
        assert b[: len(a)] == a and set(b[len(a):]) <= {"device"}, name


def test_public_names_exist(ref):
    for name in ref["names"]["top_level"]:
        assert hasattr(pm, name), name
    assert hasattr(pm.Graph, "draw") and hasattr(pm.preprocess, "generic")
    for name in ("scale", "shortest_paths", "k_nearest_neighbors", "breadth_first_order", "Graph"):
        assert hasattr(pm.preprocess.graph, name), name
    assert ref["signatures"]["preprocess.graph.shortest_paths"] == _params(pm.preprocess.graph.shortest_paths)
    assert ref["signatures"]["Graph.draw"] == _params(pm.Graph.draw)
    for mod, names in ref["names"]["modules"].items():
        o = getattr(pm, mod)
        for name in names:
            assert hasattr(o, name), "%s.%s" % (mod, name)


def test_host_helpers_agree_with_the_reference(helpers):
    h = {k: torch.from_numpy(v) for k, v in helpers.items()}
    w, d = h["w"], h["d"]
    for i, (name, args) in enumerate((("Sigmoid", (1.0, 2.0)), ("Sigmoid", (0.5,)), ("Hinge", (1.0,)),
                                      ("Hinge", (1.5, 0.2)))):
        b = getattr(pm.penalties, name)(w, *args)(d)
        assert torch.equal(h["penalty%d" % i], b), name
    np.testing.assert_allclose(pm.rotate(h["X2"], 33.0).numpy(), helpers["rotate2"], atol=1e-6)
    np.testing.assert_allclose(pm.rotate(h["X3"], h["deg"]).numpy(), helpers["rotate3"], atol=1e-6)
    with pytest.raises(ValueError):
        pm.rotate(torch.randn(4, 5), 1.0)
    assert torch.equal(pm.util.random_edges(50, 100, seed=3), h["random_edges"])
    e, wt = torch.tensor([[0, 1], [1, 3]]), torch.tensor([1.0, 2.0])
    assert abs(pm.util.adjacency_matrix(5, 2, e, wt).toarray() - helpers["adjacency"]).max() == 0
    Xq = torch.tensor([[1.0, 1.0], [1.0, -1.0], [-1.0, 1.0], [-1.0, -1.0]])  # exactly standardized
    assert pm.util.in_stdemb(Xq) and bool(helpers["Xq_in_stdemb"]) and not pm.util.in_stdemb(1.1 * Xq)
    for seed in range(4):  # same (tolerance-sensitive) verdict as the reference on arbitrary inputs
        assert pm.util.in_stdemb(h["Xs%d" % seed]) == bool(helpers["Xs%d_in_stdemb" % seed])
    a, b = helpers["pca"], pm.pca(h["Y"], 2)
    np.testing.assert_allclose(np.abs(a), (b.abs()).numpy(), rtol=1e-4, atol=1e-5)  # columns up to sign
    al = pm.align(h["pca"], h["align_target"])
    np.testing.assert_allclose(al.numpy(), helpers["align"], atol=1e-5)


def test_default_device_is_cuda_only():
    assert pm.util.get_default_device().startswith("cuda")
    with pytest.raises(ValueError):
        pm.util.set_default_device("cpu")
