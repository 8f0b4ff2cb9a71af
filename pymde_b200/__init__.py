"""pymde_b200 -- a Hopper (H100, sm_90a) native solver for Minimum-Distortion Embedding,
drop-in for the hot path of cvxgrp/pymde: MDE / .embed() / average_distortion /
preserve_neighbors / preserve_distances / penalties / losses / Centered / Standardized.

The hot path is hand-written CUDA behind a C ABI (include/mde_b200.h, libmde_b200.so);
this package is the host-side mirror of the reference's Python interface.  CUDA only."""
__version__ = "0.1.0"

from . import constraints, functions, optim, util  # noqa: F401
from .constraints import Anchored, Centered, Standardized  # noqa: F401
from .functions import losses, penalties  # noqa: F401
from .problem import MDE  # noqa: F401
from .util import align, all_edges, center, rotate, seed  # noqa: F401


def __getattr__(name):
    # recipes / preprocessing import scipy & sklearn; load them on first use
    import importlib
    if name in ("preserve_neighbors", "preserve_distances", "laplacian_embedding", "embed_new_points", "recipes"):
        recipes = importlib.import_module(__name__ + ".recipes")
        return recipes if name == "recipes" else getattr(recipes, name)
    if name in ("preprocess", "Graph"):
        preprocess = importlib.import_module(__name__ + ".preprocess")
        return preprocess if name == "preprocess" else preprocess.Graph
    if name in ("quadratic", "pca"):
        quadratic = importlib.import_module(__name__ + ".quadratic")
        return quadratic if name == "quadratic" else quadratic.pca
    raise AttributeError("module 'pymde_b200' has no attribute %r" % name)
