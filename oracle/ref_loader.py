"""TEST INFRASTRUCTURE ONLY -- loader for the UNMODIFIED reference (cvxgrp/pymde).

Imports the reference `pymde` package from the directory named by the environment variable
PYMDE_REFERENCE (a checkout of cvxgrp/pymde with its Cython extension built) or, when that is
unset, from `oracle/_ref` or `baseline/_ref` (both git-ignored; e.g. a `pip install --target` of it).  Tests never need it: what they compare against is stored
under tests/golden/ (tests/golden/make_golden.py, make_api_golden.py).

The reference eagerly imports matplotlib (pymde/__init__.py:17 ->
pymde/experiment_utils.py:1-3) and pynndescent (pymde/preprocess/data_matrix.py:116),
neither of which is installed here; plotting and approximate k-NN are outside the
hot path, so empty stub modules are registered in sys.modules before the import.  So is the Cython graph
extension `pymde.preprocess._graph` when the checkout has none built: only the graph preprocessing uses it, and the
distortion functions import and run without it.
Nothing in the product (`pymde_b200/`) may import this file.
"""
import importlib
import os
from importlib.machinery import EXTENSION_SUFFIXES
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(_HERE)
_CANDIDATES = [c for c in (os.environ.get("PYMDE_REFERENCE"), os.path.join(_REPO, "oracle", "_ref"),
                            os.path.join(_REPO, "baseline", "_ref")) if c]


def _stub(name, **attrs):
    if name in sys.modules:
        return sys.modules[name]
    try:
        return importlib.import_module(name)
    except Exception:
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        mod.__path__ = []  # behave like a package
        sys.modules[name] = mod
        return mod


def reference_root():
    for c in _CANDIDATES:
        if os.path.isdir(os.path.join(c, "pymde")):
            return c
    return None


def load_reference():
    """Return the reference `pymde` module, or None if it is not available."""
    if "pymde" in sys.modules:
        return sys.modules["pymde"]
    root = reference_root()
    if root is None:
        return None
    _stub("matplotlib")
    _stub("matplotlib.pyplot")
    _stub("matplotlib.colors")
    _stub("matplotlib.animation")
    _stub("mpl_toolkits")
    _stub("mpl_toolkits.axes_grid1", make_axes_locatable=None)
    _stub("mpl_toolkits.mplot3d")
    _stub("pynndescent")
    # a checkout whose Cython graph extension was never built: the distortion functions do not use it
    pre = os.path.join(root, "pymde", "preprocess")
    if not any(os.path.exists(os.path.join(pre, "_graph" + sfx)) for sfx in EXTENSION_SUFFIXES):
        sys.modules.setdefault("pymde.preprocess._graph", types.ModuleType("pymde.preprocess._graph"))
    sys.path.insert(0, root)
    try:
        return importlib.import_module("pymde")
    except Exception as e:  # pragma: no cover
        sys.stderr.write("reference import failed: %r\n" % (e,))
        return None
    finally:
        try:
            sys.path.remove(root)
        except ValueError:
            pass
