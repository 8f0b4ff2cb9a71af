"""Recipes for constructing MDE problems (signatures of pymde/recipes.py:103-503).

The recipes build edges / weights / deviations, pick the constraint and the initial iterate, and return a
`pymde_b200.MDE` whose `embed()` runs on the CUDA path.  `device` defaults to the current CUDA device."""
import numpy as np
import scipy.sparse
import torch

from . import constraints, preprocess, problem, quadratic, util
from .functions import losses, penalties
from .preprocess import Graph


def _remove_anchor_anchor_edges(edges, data, anchors):
    """Edges whose both ends are anchored carry no information (pymde/recipes.py:15-100)."""
    if anchors.shape[0] == 0:
        return edges, data
    a = anchors.to(edges.device)
    both = torch.isin(edges[:, 0], a) & torch.isin(edges[:, 1], a)
    return edges[~both], data[~both]


def _knn_graph_max_k(long=False):
    """mde_knn_graph_max_k(), or mde_knn_graph_long_max_k(): longer neighbour lists are assembled into a host Graph."""
    from . import _lib
    lib = _lib.load()
    return int(lib.mde_knn_graph_long_max_k() if long else lib.mde_knn_graph_max_k())


def preserve_distances(data, embedding_dim=2, loss=losses.Absolute, constraint=None, max_distances=5e7,
                       device=None, verbose=False):
    """MDE problem preserving original distances (pymde/recipes.py:103-218).  For a data matrix the pair distances
    are computed and assembled into the edge list on the device (`data_matrix.distances_device`)."""
    if not isinstance(data, (np.ndarray, torch.Tensor, Graph)) and not scipy.sparse.issparse(data):
        raise ValueError("`data` must be a np.ndarray/torch.Tensor/scipy.sparse matrix, or a pymde.Graph.")
    dev = util.cuda_device(device)
    n_items = data.n_items if isinstance(data, Graph) else data.shape[0]
    retain_fraction = max_distances / (n_items * (n_items - 1) / 2)
    if isinstance(data, Graph):
        graph = preprocess.distances(data, retain_fraction=retain_fraction, verbose=verbose, device=dev)
    else:
        graph = preprocess.data_matrix.distances_device(data, retain_fraction=retain_fraction, device=dev)
    edges = graph.edges.to(dev)
    deviations = graph.distances.to(dev)
    if constraint is None:
        constraint = constraints.Centered()
    elif isinstance(constraint, constraints._Standardized):
        deviations = preprocess.scale(deviations, constraint.natural_length(n_items, embedding_dim))
    elif isinstance(constraint, constraints.Anchored):
        edges, deviations = _remove_anchor_anchor_edges(edges, deviations, constraint.anchors)
    return problem.MDE(n_items=n_items, embedding_dim=embedding_dim, edges=edges,
                       distortion_function=loss(deviations), constraint=constraint, device=dev)


def preserve_neighbors(data, embedding_dim=2, attractive_penalty=penalties.Log1p, repulsive_penalty=penalties.Log,
                       constraint=None, n_neighbors=None, repulsive_fraction=None, max_distance=None,
                       init="quadratic", device=None, verbose=False):
    """MDE problem preserving local structure (pymde/recipes.py:221-448).  For a data matrix the neighbour graph is
    assembled on the device from the search's lists (`data_matrix.k_nearest_neighbors_device`, or
    `k_nearest_neighbors_device_long` above 64) when min(n_neighbors, n - 1) <= 256; larger n_neighbors keep the
    chunked GEMM search and the host `Graph`."""
    dev = util.cuda_device(device)
    if isinstance(data, Graph):
        n = data.n_items
    elif data.shape[0] <= 1:
        raise ValueError("The data matrix must have at least two rows.")
    else:
        n = data.shape[0]
    if n_neighbors is None:
        n_neighbors = int(max(min(15, (n * (n - 1) / 2) * 0.01 / n), 5))
    if n_neighbors > n:
        problem.LOGGER.warning("Requested n_neighbors %d > number of items %d. Setting n_neighbors to %d"
                               % (n_neighbors, n, n - 1))
        n_neighbors = n - 1
    if constraint is None:
        constraint = constraints.Centered() if repulsive_penalty is not None else constraints.Standardized()
    if isinstance(data, Graph) and max_distance is None:
        max_distance = (3 * torch.quantile(data.distances, 0.75)).item()
    if verbose:
        problem.LOGGER.info("Computing %d-nearest neighbors, with max_distance=%s" % (n_neighbors, max_distance))

    k = min(n_neighbors, n - 1)
    if isinstance(data, Graph) or k > _knn_graph_max_k(long=True):
        knn = preprocess.k_nearest_neighbors(data, k=n_neighbors, max_distance=max_distance, verbose=verbose,
                                             device=dev)
    else:
        dm = preprocess.data_matrix
        build = dm.k_nearest_neighbors_device if k <= _knn_graph_max_k() else dm.k_nearest_neighbors_device_long
        knn = build(data, n_neighbors, max_distance=max_distance, device=dev)
    edges = knn.edges.to(dev)
    weights = knn.weights.to(dev)
    if isinstance(constraint, constraints.Anchored):
        edges, weights = _remove_anchor_anchor_edges(edges, weights, constraint.anchors)

    if init == "quadratic":
        if verbose:
            problem.LOGGER.info("Computing quadratic initialization.")
        X_init = quadratic.spectral(n, embedding_dim, edges, weights, max_iter=1000, device=dev)
        if not isinstance(constraint, (constraints._Centered, constraints._Standardized)):
            constraint.project_onto_constraint(X_init, inplace=True)
    elif init == "random":
        X_init = constraint.initialization(n, embedding_dim, dev)
    else:
        raise ValueError("Unsupported value '%s' for keyword argument `init`; the supported values are "
                         "'quadratic' and 'random'." % init)

    if repulsive_penalty is not None:
        if repulsive_fraction is None:
            repulsive_fraction = 0.5 if isinstance(constraint, constraints._Standardized) else 1
        n_choose_2 = int(n * (n - 1) / 2)
        n_repulsive = min(int(repulsive_fraction * edges.shape[0]), n_choose_2 - edges.shape[0])
        negative_edges = preprocess.sample_edges(n, n_repulsive, exclude=edges, device=dev).to(dev)
        negative_weights = -torch.ones(negative_edges.shape[0], dtype=X_init.dtype, device=dev)
        if isinstance(constraint, constraints.Anchored):
            negative_edges, negative_weights = _remove_anchor_anchor_edges(negative_edges, negative_weights,
                                                                           constraint.anchors)
        edges = torch.cat([edges, negative_edges])
        weights = torch.cat([weights, negative_weights])
        f = penalties.PushAndPull(weights, attractive_penalty=attractive_penalty,
                                  repulsive_penalty=repulsive_penalty)
    else:
        f = attractive_penalty(weights)

    mde = problem.MDE(n_items=n, embedding_dim=embedding_dim, edges=edges, distortion_function=f,
                      constraint=constraint, device=dev)
    mde._X_init = X_init.to(dev).float().contiguous()
    d = mde.distances(mde._X_init)
    if bool((d == 0).any()):  # overlapping points make E non-differentiable: perturb (recipes.py:438-447)
        mde._X_init = mde._X_init + 1e-4 * torch.randn_like(mde._X_init)
    return mde


def laplacian_embedding(data, embedding_dim=2, n_neighbors=None, max_distance=None, init="quadratic",
                        device=None, verbose=False):
    """Quadratic penalties + standardization on the k-NN graph (pymde/recipes.py:451-503)."""
    return preserve_neighbors(data, embedding_dim=embedding_dim, attractive_penalty=penalties.Quadratic,
                              repulsive_penalty=None, n_neighbors=n_neighbors, max_distance=max_distance,
                              init=init, device=device, verbose=verbose)
