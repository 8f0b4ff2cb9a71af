"""Host-side utilities of the CUDA MDE path (API surface of pymde/util.py kept where it matters).

Everything numerical here is CUDA-only: tensors must live on a CUDA device; there is no CPU
fallback for the hot path (pymde_b200._lib raises if the extension is missing)."""
import numbers

import numpy as np
import torch

from . import _lib

_NP_RNG = np.random.default_rng()
_DEFAULT_DEVICE = "cuda"  # see get_default_device / set_default_device


class SolverError(Exception):
    """Raised where the reference raises pymde.util.SolverError (pymde/util.py:16)."""


def cuda_device(device=None):
    """Canonical CUDA device.  None -> current CUDA device.  CPU devices are rejected loudly."""
    if device is None:
        device = _DEFAULT_DEVICE
    dev = torch.device(device) if not isinstance(device, torch.device) else device
    if dev.type != "cuda":
        raise ValueError(
            "pymde_b200 runs the MDE hot path on CUDA (sm_90a) only; got device %r. "
            "There is no CPU fallback." % (device,))
    if not torch.cuda.is_available():
        raise RuntimeError("pymde_b200 needs a CUDA device (torch.cuda.is_available() is False)")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def stream_ptr(device):
    return torch.cuda.current_stream(device).cuda_stream


def _is_numeric(arg):
    return isinstance(arg, (numbers.Number, np.ndarray, np.generic, torch.Tensor))


def to_tensor(args, device=None):
    """Numbers / ndarrays -> torch tensors (float64 ndarrays become float32, as in pymde/util.py:59-78)."""
    single = not isinstance(args, (list, tuple))
    seq = [args] if single else list(args)
    out = []
    for a in seq:
        if isinstance(a, torch.Tensor):
            out.append(a)
        elif _is_numeric(a):
            if isinstance(a, np.ndarray) and a.dtype == np.float64:
                out.append(torch.tensor(a, dtype=torch.float32, device=device))
            else:
                out.append(torch.tensor(a, device=device))
        else:
            raise ValueError("Received non-numeric argument ", a)
    return out[0] if single else out


def as_f32_cuda(t, device):
    """Contiguous float32 CUDA copy/view of a tensor-like."""
    t = to_tensor(t)
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def all_edges(n):
    """All (n choose 2) edges (pymde/util.py:103-117)."""
    return torch.triu_indices(n, n, 1).T


def natural_length(n, m):
    return torch.sqrt(torch.tensor(2.0 * n * m / (n - 1)))


def np_rng():
    return _NP_RNG


def seed(seed: int):
    """Seed torch, numpy's legacy global state and the module Generator (pymde/util.py:398-408)."""
    global _NP_RNG
    torch.manual_seed(seed)
    np.random.seed(seed)
    _NP_RNG = np.random.default_rng(seed)


def center(X):
    X = to_tensor(X)
    return X - X.mean(dim=0)[None, :]


def procrustes(X_source, X_target):
    """argmin_Q |X_source Q - X_target|_F over orthogonal Q (pymde/util.py:200-205)."""
    U, _, Vh = torch.linalg.svd(X_target.T @ X_source, full_matrices=False)
    return Vh.transpose(-2, -1) @ U.T


def align(source, target):
    """Rotate `source` onto `target` (orthogonal Procrustes; pymde/util.py:290-331)."""
    source, target = to_tensor(source), to_tensor(target)
    mu = source.mean(dim=0)
    src = source - mu[None, :]
    rms = src.norm(dim=0)
    src = src / rms[None, :]
    tgt = center(target)
    tgt = tgt / tgt.norm(dim=0)
    Q = procrustes(src, tgt)
    return (src @ Q) * rms[None, :] + mu


def rotate(X, degrees):
    """Rotate a 2-D embedding by `degrees` (scalar) or a 3-D one by three angles: about the x axis first, then
    y, then z (pymde/util.py:255-288; row vectors, X @ R)."""
    X = to_tensor(X)
    degrees = to_tensor(degrees).to(X.device)
    if X.shape[1] not in (2, 3):
        raise ValueError("Only 2 or 3 dimensional embeddings can be rotated using this method.")
    rad = torch.deg2rad(degrees.float().reshape(-1))
    c, s = torch.cos(rad), torch.sin(rad)
    if X.shape[1] == 2:
        if rad.numel() != 1:
            raise ValueError("`degrees` must be a scalar.")
        R = torch.stack([torch.stack([c[0], -s[0]]), torch.stack([s[0], c[0]])])
        return X @ R.to(X.dtype)
    if rad.numel() != 3:
        raise ValueError("`degrees` must be a length-3 tensor.")
    one, zero = torch.ones_like(c[0]), torch.zeros_like(c[0])
    Rx = torch.stack([torch.stack([one, zero, zero]), torch.stack([zero, c[0], s[0]]), torch.stack([zero, -s[0], c[0]])])
    Ry = torch.stack([torch.stack([c[1], zero, -s[1]]), torch.stack([zero, one, zero]), torch.stack([s[1], zero, c[1]])])
    Rz = torch.stack([torch.stack([c[2], s[2], zero]), torch.stack([-s[2], c[2], zero]), torch.stack([zero, zero, one])])
    return X @ (Rx @ Ry @ Rz).to(X.dtype)


def in_stdemb(X):
    """True when X is centered with (1/n) X^T X = I (pymde/util.py:121-126; any embedding dimension here)."""
    X = to_tensor(X)
    cov = (1.0 / X.shape[0]) * X.T @ X
    eye = torch.eye(X.shape[1], dtype=X.dtype, device=X.device)
    return bool(torch.isclose(cov, eye).all() and torch.isclose(X.mean(dim=0), torch.zeros_like(cov[0])).all())


def random_edges(n, p, seed=0):
    """p distinct uniformly random pairs i < j (pymde/util.py:411-422): indices into the row-major upper
    triangle drawn without replacement, mapped back to (i, j) by the closed-form inverse."""
    n, p = int(n), int(p)
    idx = np.random.default_rng(seed).choice(n * (n - 1) // 2, p, replace=False, shuffle=False).astype(np.float64)
    i = n - 2 - np.floor(np.sqrt(-8.0 * idx + 4.0 * n * (n - 1) - 7.0) / 2.0 - 0.5)
    j = idx + i + 1 - n * (n - 1) / 2 + (n - i) * ((n - i) - 1) / 2
    return torch.tensor(np.stack([i, j], axis=1).astype(np.int64))


def adjacency_matrix(n, m, edges, weights, use_scipy=True):
    """Symmetric weighted adjacency matrix A + A^T of the edge list (pymde/util.py:174-198); `m` is unused, as in
    the reference.  scipy COO by default, torch sparse COO otherwise."""
    del m
    if use_scipy:
        import scipy.sparse
        w = weights.detach().cpu().numpy() if isinstance(weights, torch.Tensor) else np.asarray(weights)
        e = edges.detach().cpu().numpy() if isinstance(edges, torch.Tensor) else np.asarray(edges)
        A = scipy.sparse.coo_matrix((w, (e[:, 0], e[:, 1])), shape=(n, n), dtype=np.float32)
        return (A + A.T).tocoo()
    A = torch.sparse_coo_tensor(edges.transpose(0, 1), weights, size=(n, n), dtype=torch.float32, device=edges.device)
    return A + A.transpose(0, 1)


def get_default_device():
    """Device recipes use when none is given (pymde/util.py:20-37).  Always a CUDA device here."""
    return str(_DEFAULT_DEVICE)


def set_default_device(device):
    global _DEFAULT_DEVICE
    dev = torch.device(device) if not isinstance(device, torch.device) else device
    if dev.type != "cuda":
        raise ValueError("pymde_b200 runs on CUDA devices only; got %r" % (device,))
    _DEFAULT_DEVICE = dev


def scale_delta(delta, d_nat):
    delta = to_tensor(delta)
    rms = torch.sqrt(torch.mean(delta.float() ** 2))
    return delta * float(d_nat) / rms


class Workspace(object):
    """Per-device scratch tensors handed to the C ABI (projection workspace, loss accumulator)."""
    _cache = {}

    @classmethod
    def get(cls, device, nbytes):
        key = (str(device),)
        buf = cls._cache.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(int(nbytes), 1 << 16), dtype=torch.uint8, device=device)
            cls._cache[key] = buf
        return buf


def proj_standardized(X, demean=False, inplace=False):
    """sqrt(n) * polar factor of X (pymde/util.py:129-171), on the device.

    m <= 32: fused Gram + on-device Jacobi kernels; 32 < m <= 256: tiled Gram, Newton-Schulz inverse square root
    and row kernel (csrc/mde_project_wide.cu) -- both behind mde_project_standardized.  Larger m: the same Gram /
    eigen formulation with the m x m eigenproblem handed to cuSOLVER through torch."""
    if X.device.type != "cuda":
        raise ValueError("pymde_b200.util.proj_standardized needs a CUDA tensor")
    out = X if inplace else X.detach().clone()
    if out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("expected a contiguous float32 tensor")
    n, m = out.shape
    lib = _lib.load()
    if m <= 256 and demean:
        ws = Workspace.get(out.device, lib.mde_project_ws_bytes(n, m))
        _lib.check(lib.mde_project_standardized(out.data_ptr(), n, m, ws.data_ptr(), stream_ptr(out.device)))
        return out
    with torch.no_grad():
        Z = out.double()
        if demean:
            Z = Z - Z.mean(dim=0)
        lam, Q = torch.linalg.eigh(Z.T @ Z)
        if not bool((lam > 0).all()):
            raise SolverError("Gram matrix is not positive definite")
        W = (Q * lam.rsqrt()) @ Q.T * (float(n) ** 0.5)
        out.copy_((Z @ W).float())
    return out
