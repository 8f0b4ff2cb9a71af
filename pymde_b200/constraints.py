"""Constraint sets (interface of pymde/constraints.py:7-254), backed by the CUDA projection kernels.

`Centered()` / `Standardized()` return module-level singletons like the reference
(pymde/constraints.py:234-254); recipes detect them with isinstance(c, _Standardized)."""
import abc

import torch

from . import _lib
from . import util


class Constraint(abc.ABC):
    """A generic constraint.  Subclass and implement the four methods to create your own;
    custom constraints run through the generic (torch-tensor) solver in pymde_b200.optim, or, under
    PYMDE_B200_CONSTRAINT=device, inside the device-resident solver's steps (pymde_b200/external.py)."""

    @abc.abstractmethod
    def name(self) -> str:
        raise NotImplementedError

    @abc.abstractmethod
    def initialization(self, n_items: int, embedding_dim: int, device=None) -> torch.Tensor:
        raise NotImplementedError

    @abc.abstractmethod
    def project_onto_constraint(self, Z: torch.Tensor, inplace=True) -> torch.Tensor:
        raise NotImplementedError

    @abc.abstractmethod
    def project_onto_tangent_space(self, X: torch.Tensor, Z: torch.Tensor, inplace=True) -> torch.Tensor:
        raise NotImplementedError


def _check(Z):
    if Z.device.type != "cuda":
        raise ValueError("pymde_b200 constraints operate on CUDA tensors only (got %s)" % Z.device)
    if Z.dtype != torch.float32 or not Z.is_contiguous() or Z.dim() != 2:
        raise ValueError("expected a contiguous float32 (n, m) tensor")


def _ws(Z):
    lib = _lib.load()
    n, m = Z.shape
    return util.Workspace.get(Z.device, lib.mde_project_ws_bytes(n, m))


class _Centered(Constraint):
    _solver_id = _lib.CONSTRAINT_CENTERED

    def name(self):
        return "centered"

    def initialization(self, n_items, embedding_dim, device=None):
        dev = util.cuda_device(device)
        X = torch.randn((int(n_items), int(embedding_dim)), device=dev)
        return self.project_onto_constraint(X, inplace=True)

    def project_onto_tangent_space(self, X, Z, inplace=True):
        del X
        return Z

    def project_onto_constraint(self, Z, inplace=True):
        out = Z if inplace else Z.detach().clone()
        _check(out)
        n, m = out.shape
        lib = _lib.load()
        _lib.check(lib.mde_project_centered(out.data_ptr(), n, m, _ws(out).data_ptr(), util.stream_ptr(out.device)))
        return out


class Anchored(Constraint):
    """Anchor some vectors to specific values (pymde/constraints.py:114-164)."""
    _solver_id = _lib.CONSTRAINT_ANCHORED

    def __init__(self, anchors, values):
        super(Anchored, self).__init__()
        self.anchors = anchors
        self.values = values

    def name(self):
        return "anchored"

    def initialization(self, n_items, embedding_dim, device=None):
        dev = util.cuda_device(device)
        X = torch.randn((int(n_items), int(embedding_dim)), device=dev)
        X[self.anchors.to(dev)] = self.values.to(dev)
        return X

    def project_onto_tangent_space(self, X, Z, inplace=True):
        del X
        out = Z if inplace else Z.detach().clone()
        out[self.anchors.to(out.device), :] = 0.0
        return out

    def project_onto_constraint(self, Z, inplace=True):
        out = Z if inplace else Z.detach().clone()
        out[self.anchors.to(out.device), :] = self.values.to(out.device)
        return out


class _Standardized(Constraint):
    """Centered and (1/n) X^T X = I."""
    _solver_id = _lib.CONSTRAINT_STANDARDIZED

    def name(self):
        return "standardized"

    def initialization(self, n_items, embedding_dim, device=None):
        dev = util.cuda_device(device)
        X = torch.randn((int(n_items), int(embedding_dim)), device=dev)
        return self.project_onto_constraint(X, inplace=True)

    def project_onto_tangent_space(self, X, Z, inplace=True):
        out = Z if inplace else Z.detach().clone()
        _check(out)
        _check(X)
        n, m = out.shape
        if m <= 1024:
            lib = _lib.load()
            _lib.check(lib.mde_tangent_standardized(X.data_ptr(), out.data_ptr(), n, m, _ws(out).data_ptr(),
                                                    util.stream_ptr(out.device)))
            return out
        with torch.no_grad():  # m > 1024: plain library GEMMs for the m x m product
            gtx = out.T @ X
            out.sub_((1.0 / n) * (X @ gtx))
        return out

    def project_onto_constraint(self, Z, inplace=True):
        return util.proj_standardized(Z, demean=True, inplace=inplace)

    def natural_length(self, n_items, embedding_dim):
        return (torch.tensor(2.0) * n_items * embedding_dim / (n_items - 1)).sqrt()


__Centered = _Centered()
__Standardized = _Standardized()


def is_builtin(constraint):
    """Is `constraint` one the device solver projects with its own kernels (not a user-defined subclass)?"""
    return type(constraint) in (_Centered, _Standardized, Anchored)


def Centered():
    """Centering constraint (singleton): embedding vectors have mean zero."""
    return __Centered


def Standardized():
    """Standardization constraint (singleton): centered and (1/n) X^T X = I."""
    return __Standardized
