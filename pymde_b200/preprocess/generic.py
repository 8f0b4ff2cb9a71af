"""Type dispatch between data matrices and graphs (interface of pymde/preprocess/generic.py:13-108)."""
from . import data_matrix, graph
from .graph import Graph


def _graph_on_device(A):
    """Graph searches run on the device (bit-parallel BFS or the batched Bellman-Ford engine, DESIGN section 10)
    unless the graph is tiny or PYMDE_B200_SHORTEST_PATHS=host asks for scipy's Dijkstra."""
    import os
    import torch
    return (torch.cuda.is_available() and A.shape[0] > 256
            and os.environ.get("PYMDE_B200_SHORTEST_PATHS", "device") != "host")


def distances(data, retain_fraction=1.0, verbose=False, device=None):
    """Distances between the items of `data` (a matrix of row vectors or a Graph) as a Graph: Euclidean distances
    of all pairs / a uniform sample of them, or shortest-path lengths."""
    if isinstance(data, Graph):
        if _graph_on_device(data.adjacency_matrix):
            return graph.shortest_paths_device(data, retain_fraction=retain_fraction, device=device)
        return graph.shortest_paths(data, retain_fraction=retain_fraction, verbose=verbose)
    return data_matrix.distances(data, retain_fraction=retain_fraction, verbose=verbose, device=device)


def k_nearest_neighbors(data, k, max_distance=None, verbose=False, device=None):
    """k-nearest-neighbour graph of `data` (Euclidean for matrices, shortest-path metric for graphs)."""
    if isinstance(data, Graph):
        if _graph_on_device(data.adjacency_matrix) and k <= _graph_knn_max_k():
            return graph.k_nearest_neighbors_device(data, k, max_distance=max_distance, device=device)
        return graph.k_nearest_neighbors(data, k, max_distance=max_distance, verbose=verbose)
    return data_matrix.k_nearest_neighbors(data, k, max_distance=max_distance, verbose=verbose, device=device)


def _graph_knn_max_k():
    from .. import _lib
    return int(_lib.load().mde_graph_knn_max_k())
