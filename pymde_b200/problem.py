"""Minimum-Distortion Embedding problem object (API of pymde/problem.py:36-527).

`MDE` keeps the reference's constructor, attributes and methods.  The bodies of
`average_distortion`, `distances`, `distortions` and `embed` dispatch to the CUDA path:
the (p,2) int64 edge list is narrowed / sorted once into a device-resident layout
(`mde_edges_create`), every evaluation is ONE fused forward+backward kernel
(`mde_distortion`), and `embed` hands the whole projected L-BFGS solve to the device
(`pymde_b200.optim.lbfgs` -> `mde_solver_*`).  CUDA only: there is no CPU fallback."""
import ctypes as C
import logging
import sys
import typing as tp

import torch

from . import _lib
from . import constraints
from . import optim
from . import util
from .functions.function import Function

LOGGER = logging.getLogger("__pymde_b200__")
LOGGER.propagate = False
LOGGER.setLevel(logging.INFO)
if not LOGGER.handlers:
    _h = logging.StreamHandler(sys.stdout)
    _h.setLevel(logging.INFO)
    _h.setFormatter(logging.Formatter(fmt="%(asctime)s: %(message)s", datefmt="%b %d %I:%M:%S %p"))
    LOGGER.addHandler(_h)


class EdgeLayout(object):
    """Owner of one `mde_edges_t` (device-resident sorted int32 COO + permuted parameters)."""

    def __init__(self, edges, n_items, table, par0, par1, device, p_total=None, embedding_dim=2):
        lib = _lib.load()
        self.lib = lib
        self.device = device
        self.p = int(edges.shape[0])
        self.n = int(n_items)
        self._keep = (edges,)  # not referenced by the library after creation; kept for clarity
        par0 = util.as_f32_cuda(par0, device).reshape(-1)
        if par0.numel() == 1:
            par0 = par0.expand(self.p).contiguous()
        if par0.numel() != self.p:
            raise ValueError("distortion function has %d parameters for %d edges" % (par0.numel(), self.p))
        p1 = None
        if par1 is not None:
            p1 = util.as_f32_cuda(par1, device).reshape(-1)
            if p1.numel() == 1:
                p1 = p1.expand(self.p).contiguous()
        e = edges.to(device=device, dtype=torch.int64).contiguous()
        handle = C.c_void_p()
        self.table = table
        with torch.cuda.device(device):
            _lib.check(lib.mde_edges_create_ex(C.byref(handle), e.data_ptr(), self.p, self.n, par0.data_ptr(),
                                               None if p1 is None else p1.data_ptr(), C.byref(table),
                                               int(self.p if p_total is None else p_total), int(embedding_dim),
                                               util.stream_ptr(device)))
        self.handle = handle
        self.loss = torch.zeros(1, dtype=torch.float64, device=device)
        self.p_total = int(self.p if p_total is None else p_total)
        self.dist = None  # set by MDE._layout() for an edge shard: evaluations are summed across ranks

    def close(self):
        if getattr(self, "handle", None):
            self.lib.mde_edges_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def value_and_grad(self, X, want_grad=True):
        """(sum_k f_k as a float64 0-dim tensor / p_total, grad (n,m) or None).  One fused launch."""
        n, m = X.shape
        grad = torch.zeros_like(X) if want_grad else None
        self.loss.zero_()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mde_distortion(self.handle, X.data_ptr(), m,
                                               None if grad is None else grad.data_ptr(),
                                               self.loss.data_ptr(), util.stream_ptr(self.device)))
        if self.dist is not None:
            from . import dist as pdist
            pdist.allreduce_evaluation(self.loss, grad, self.dist.get("group"))
        value = (self.loss[0] / self.p_total).to(torch.float32)
        return value, grad

    def outputs(self, X, distances=True, distortions=False):
        n, m = X.shape
        d = torch.empty(self.p, dtype=torch.float32, device=self.device) if distances else None
        f = torch.empty(self.p, dtype=torch.float32, device=self.device) if distortions else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mde_edge_outputs(self.handle, X.data_ptr(), m,
                                                 None if d is None else d.data_ptr(),
                                                 None if f is None else f.data_ptr(),
                                                 util.stream_ptr(self.device)))
        return d, f

    def scatter_external(self, X, g):
        grad = torch.zeros_like(X)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mde_scatter_external(self.handle, X.data_ptr(), X.shape[1], g.data_ptr(),
                                                     grad.data_ptr(), util.stream_ptr(self.device)))
        if self.dist is not None:
            import torch.distributed as tdist
            tdist.all_reduce(grad, op=tdist.ReduceOp.SUM, group=self.dist.get("group"))
        return grad


class _FusedAverageDistortion(torch.autograd.Function):
    """Seam of pymde/average_distortion.py:36-83: forward returns the 0-dim average distortion;
    when X requires grad the gradient is produced by the same launch and kept for backward,
    which honours grad_output scaling (:79); otherwise nothing is saved (:64-65)."""

    @staticmethod
    def forward(ctx, X, layout):
        want = X.requires_grad
        value, grad = layout.value_and_grad(X.detach(), want_grad=want)
        if want:
            ctx.save_for_backward(grad)
        return value

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        return grad * grad_output, None


class _ExternalAverageDistortion(torch.autograd.Function):
    """Arbitrary Python callables as distortion functions (seam #4): distances and the
    scatter run on the CUDA kernels, only f itself is the user's torch code."""

    @staticmethod
    def forward(ctx, X, layout, f):
        Xd = X.detach()
        norms, _ = layout.outputs(Xd, distances=True)

        def mean(values):  # global mean: an edge shard divides by the global edge count and sums across ranks
            if layout.dist is None:
                return values.mean()
            return values.sum() / layout.p_total

        def reduced(value):
            if layout.dist is not None:
                import torch.distributed as tdist
                value = value.clone()
                tdist.all_reduce(value, op=tdist.ReduceOp.SUM, group=layout.dist.get("group"))
            return value

        if X.requires_grad:
            with torch.enable_grad():
                norms.requires_grad_(True)
                distortion = mean(f(norms))
                distortion.backward()
                norms.requires_grad_(False)
            g = norms.grad / norms
            g[~torch.isfinite(g)] = 1.0
            ctx.save_for_backward(layout.scatter_external(Xd, g.contiguous()))
            return reduced(distortion.detach())
        return reduced(mean(f(norms)))

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        return grad * grad_output, None, None


class MDE(torch.nn.Module):
    """An MDE problem: n_items, embedding_dim, edges, a vector distortion function and a
    constraint (pymde/problem.py:36-193).  Tensors live on a CUDA device."""

    def __init__(self, n_items: int, embedding_dim: int, edges: torch.Tensor,
                 distortion_function: tp.Callable, constraint: tp.Optional[constraints.Constraint] = None,
                 device: tp.Optional[str] = None):
        super(MDE, self).__init__()
        if device is None and isinstance(edges, torch.Tensor) and edges.device.type == "cuda":
            device = edges.device
        self.device = util.cuda_device(device)

        if not isinstance(n_items, torch.Tensor):
            n_items = torch.tensor(int(n_items), device=self.device)
        self.register_buffer("n_items", n_items.to(self.device))
        if not isinstance(embedding_dim, torch.Tensor):
            embedding_dim = torch.tensor(int(embedding_dim), device=self.device)
        self.register_buffer("embedding_dim", embedding_dim.to(self.device))

        if edges is None:
            raise ValueError("edges are required (stochastic functions are not part of the CUDA path)")
        if not isinstance(edges, torch.Tensor):
            edges = torch.tensor(edges, dtype=torch.int64, device=self.device)
        if edges.dim() != 2 or edges.shape[1] != 2:
            raise ValueError("edges must have shape (num_edges, 2)")
        self_edges = edges[:, 0] == edges[:, 1]
        if bool(self_edges.any()):
            offending = torch.where(self_edges)[0]
            raise ValueError("The edge list must not contain self edges; the following rows were found "
                             "to be self edges: ", offending.cpu().numpy())
        if str(edges.device) != str(self.device):
            edges = edges.to(self.device)
        if edges.dtype != torch.int64:
            edges = edges.long()
        p = torch.tensor(edges.shape[0], device=self.device)
        n = int(self.n_items)
        complete = n * (n - 1) // 2
        if int(p) > complete:
            raise ValueError("Your graph has more than (n_items choose 2) edges."
                             "(p: {0}, n_items choose 2: {1})".format(int(p), complete))
        if int(edges.min()) < 0 or int(edges.max()) >= n:
            raise ValueError("edge endpoints must lie in [0, n_items)")
        self.register_buffer("edges", edges)
        self.register_buffer("p", p)
        self.register_buffer("_complete_graph_edges", torch.tensor(complete, device=self.device))

        if isinstance(distortion_function, torch.nn.Module):
            f_dev = getattr(distortion_function, "device", None)
            if f_dev is None or str(f_dev) != str(self.device):
                distortion_function = distortion_function.to(self.device)
        self.distortion_function = distortion_function
        if constraint is None:
            constraint = constraints.Centered()
        self.constraint = constraint

        self.register_buffer("X", None)
        self.register_buffer("_X_init", None)
        self.solve_stats = None
        self.value = None
        self.residual_norm = None
        self.__dict__["_edge_layout"] = None
        self.__dict__["_device_solver"] = None
        self.__dict__["_dist"] = None  # (rank, world_size, allreduce) for edge-sharded solves

    # ------------------------------------------------------------------------------------
    def __str__(self):
        f = self.distortion_function
        fname = f.__name__ if hasattr(f, "__name__") else type(f).__name__
        return ("MDE problem:\n\tn (number of items) {0}\n\tm (embedding dimension) {1}\n"
                "\tp (number of edges) {2}\n\tfraction of total edges {3:.1e}\n"
                "\t{4} distortion functions\n\tconstraint {5}\n\tdevice {6}".format(
                    int(self.n_items), int(self.embedding_dim), int(self.p),
                    float(self.p) / max(int(self._complete_graph_edges), 1), fname,
                    self.constraint.name(), self.device))

    def _repr_pretty_(self, p, cycle):
        del cycle
        p.text(self.__str__())

    # ---- CUDA path plumbing ------------------------------------------------------------------
    def __setattr__(self, name, value):
        # the layout snapshots the distortion function's parameters, the device solver the constraint's:
        # replacing either must not leave stale device copies behind (the reference re-reads them every evaluation)
        if name in ("distortion_function", "constraint") and "_edge_layout" in self.__dict__:
            self._invalidate(layout=(name == "distortion_function"))
        super(MDE, self).__setattr__(name, value)

    def _invalidate(self, layout=True):
        cur = self.__dict__.get("_device_solver")
        if cur is not None:
            cur[1].close()
            self.__dict__["_device_solver"] = None
        if layout:
            lay = self.__dict__.get("_edge_layout")
            if lay is not None:
                lay.close()
                self.__dict__["_edge_layout"] = None

    @staticmethod
    def _tensor_stamp(*tensors):
        """(data_ptr, in-place version, shape) of every tensor: changes when a parameter is mutated or replaced."""
        return tuple((int(t.data_ptr()), int(t._version), tuple(t.shape)) for t in tensors if isinstance(t, torch.Tensor))

    def _function_stamp(self):
        if not self._is_table_function():
            return ("external", id(self.distortion_function))
        table, par0, par1 = self.distortion_function._table()
        scal = (table.fn_att, table.fn_rep, tuple(table.att), tuple(table.rep), table.push_pull)
        return (scal,) + self._tensor_stamp(par0, par1)

    def _is_table_function(self):
        f = self.distortion_function
        return isinstance(f, Function) and f._supported()

    def _layout(self):
        lay = self.__dict__["_edge_layout"]
        if lay is not None and lay.stamp != self._function_stamp():
            self._invalidate(layout=True)  # weights / deviations / scalars were mutated since the layout was built
            lay = None
        if lay is None:
            if self._is_table_function():
                table, par0, par1 = self.distortion_function._table()
            else:  # external callable: the layout only needs the index structure
                table = _lib.mde_fn_t()
                table.fn_att = table.fn_rep = 100
                par0, par1 = torch.zeros(int(self.p), device=self.device), None
            p_total = None if self.__dict__["_dist"] is None else self.__dict__["_dist"]["p_total"]
            lay = EdgeLayout(self.edges, int(self.n_items), table, par0, par1, self.device, p_total=p_total,
                             embedding_dim=int(self.embedding_dim))
            lay.dist = self.__dict__["_dist"]
            lay.stamp = self._function_stamp()
            self.__dict__["_edge_layout"] = lay
        return lay

    def _fused_ok(self, constraint, memory_size):
        """Can the device-resident solver take this problem?  Table functions and callables alike; callables of
        edge-sharded problems, and callables under PYMDE_B200_EXTERNAL=generic, stay on the host-stepped solver.
        User-defined constraints run on it only under PYMDE_B200_CONSTRAINT=device|graph|hook, on one GPU."""
        from . import external
        if not self._is_table_function():
            if not callable(self.distortion_function) or self.__dict__["_dist"] is not None:
                return False
            if external.forced_mode() == "generic":
                return False
        if not constraints.is_builtin(constraint):
            if external.constraint_mode() is None or self.__dict__["_dist"] is not None:
                return False
        m = int(self.embedding_dim)
        if (m % 4 == 0 and m > 1024) or (m % 4 != 0 and m > 512):  # mirrors launch_distortion (mde_edges.cu)
            return False
        return 1 <= int(memory_size) <= 32

    def _solver(self, constraint, memory_size, max_iter, external=None, constraint_part=None):
        """Device solver for this problem, cached across embed() calls.  `max_iter` only sizes the statistics
        buffers, so a cached solver with enough capacity is reused (its CUDA graphs are built once, except for a
        callable distortion function or a user-defined constraint: `external` and `constraint_part`, their newly
        captured parts, are installed and the graphs rebuilt)."""
        layout = self._layout()  # (re)built first: a rebuilt layout invalidates the solver that referenced the old one
        stamp = ()
        if isinstance(constraint, constraints.Anchored):  # anchor indices / values are copied at solver creation
            stamp = self._tensor_stamp(constraint.anchors, constraint.values)
        key = (int(memory_size), stamp)
        cur = self.__dict__["_device_solver"]
        if cur is None or cur[2] is not constraint or cur[0] != key or cur[1].max_iter < int(max_iter):
            if cur is not None:
                cur[1].close()
            dist = self.__dict__["_dist"]
            capacity = max(int(max_iter), 1024)
            solver = optim.DeviceSolver(layout, int(self.n_items), int(self.embedding_dim), constraint,
                                        memory_size, capacity,
                                        world_size=1 if dist is None else dist["world_size"],
                                        allreduce=None if dist is None else dist.get("allreduce"),
                                        exchange=None if dist is None else dist.get("exchange"),
                                        rank=0 if dist is None else dist["rank"], external=external,
                                        constraint_part=constraint_part)
            cur = (key, solver, constraint)  # holds the constraint: a recycled id() can never alias it
            self.__dict__["_device_solver"] = cur
        else:
            if external is not None:
                cur[1].set_external(external)
            if constraint_part is not None:
                cur[1].set_constraint_part(constraint_part)
        return cur[1]

    def _check_X(self, X):
        if X is None:
            X = self.X
        if X is None:
            raise ValueError("Call this function after running the `embed` method, or provide a value "
                             "for the embedding argument `X`")
        if X.device.type != "cuda":
            raise ValueError("pymde_b200 evaluates CUDA tensors only; move X to %s" % (self.device,))
        if X.dtype != torch.float32:
            raise ValueError("the CUDA path computes in float32; got %s" % X.dtype)
        if not X.is_contiguous():
            return X.contiguous()
        # the kernels load a row of m = 2 as one float2 and rows of m % 4 == 0 as float4s: a contiguous view that
        # starts inside a row of its storage (e.g. buf[1:].view(n, m)) is copied to storage aligned for those loads
        m = X.shape[1] if X.dim() == 2 else 1
        align = 16 if m % 4 == 0 else (8 if m == 2 else 4)
        if X.data_ptr() % align != 0:
            return X.clone(memory_format=torch.contiguous_format)
        return X

    # ---- evaluation API ---------------------------------------------------------------------
    def differences(self, X):
        """X[i] - X[j] for each edge (i, j)."""
        return X[self.edges[:, 0]] - X[self.edges[:, 1]]

    def distances(self, X=None):
        """Embedding distances, one per edge, in the order of `self.edges` (problem.py:252-279)."""
        X = self._check_X(X)
        d, _ = self._layout().outputs(X.detach(), distances=True)
        return d

    def distortions(self, X=None):
        """Distortions f_k(d_k), one per edge (problem.py:281-307)."""
        X = self._check_X(X)
        if self._is_table_function():
            _, f = self._layout().outputs(X.detach(), distances=False, distortions=True)
            return f
        return self.distortion_function(self.distances(X))

    def average_distortion(self, X=None):
        """Average distortion as a 0-dim tensor with autograd support (problem.py:309-336)."""
        X = self._check_X(X)
        if self._is_table_function():
            return _FusedAverageDistortion.apply(X, self._layout())
        return _ExternalAverageDistortion.apply(X, self._layout(), self.distortion_function)

    def high_distortion_pairs(self, X=None):
        """Edges and distortions sorted from high to low distortion (problem.py:338-384)."""
        distortions = self.distortions(X)
        idx = torch.argsort(distortions, descending=True, stable=True)
        return self.edges[idx], distortions[idx]

    # ---- solve ------------------------------------------------------------------------------
    def embed(self, X=None, eps=1e-5, max_iter=300, memory_size=10, verbose=False, print_every=None,
              snapshot_every=None):
        """Compute an embedding (problem.py:386-527); stores it in `self.X`, statistics in
        `self.solve_stats`, and returns it."""
        if X is None and self._X_init is not None:
            X = self._X_init.detach().clone()
        elif X is None:
            X = self.constraint.initialization(self.n_items, self.embedding_dim, self.device)
        else:
            X = X.detach().clone()
        if X.device != self.device:
            X = X.to(self.device)  # host -> device copy of the initial iterate
        X = X.to(torch.float32).contiguous()
        if max_iter < 0:
            raise ValueError("`max_iter` must be greater than 0")
        if memory_size <= 0:
            raise ValueError("`memory_size` must be greater than 0")
        if verbose:
            LOGGER.info("Fitting a %s embedding into R^%d, for a graph with %d items and %d edges." % (
                self.constraint.name(), int(self.embedding_dim), int(self.n_items), int(self.p)))
            LOGGER.info("`embed` method parameters: eps=%.1e, max_iter=%d, memory_size=%d" % (
                eps, max_iter, memory_size))
        if print_every is None:
            print_every = max(1, max_iter // 10)

        X_star, solve_stats = optim.lbfgs(
            X=X, constraint=self.constraint, objective_fn=self.average_distortion, eps=eps, max_iter=max_iter,
            memory_size=memory_size, use_line_search=True, use_cached_loss=True, verbose=verbose,
            print_every=print_every, snapshot_every=snapshot_every, logger=LOGGER)

        self.X = X_star
        self.solve_stats = solve_stats
        if solve_stats.iterations:
            self.value = solve_stats.average_distortions[-1]
            self.residual_norm = solve_stats.residual_norms[-1]
        if verbose:
            LOGGER.info("Finished fitting in %.3f seconds and %d iterations." % (
                solve_stats.solve_time, solve_stats.iterations))
            if solve_stats.iterations:
                LOGGER.info("average distortion %.3g | residual norm %.1e" % (self.value, self.residual_norm))
        return self.X

    forward = embed

    # visualisation is outside the hot path (SURVEY section 2 row 19)
    def plot(self, *args, **kwargs):
        raise NotImplementedError("plotting is out of scope for pymde_b200; use pymde.plot on mde.X.cpu()")

    play = plot
    distortions_cdf = plot
