"""Solve driver (interface of pymde/optim.py:11-184).

`lbfgs(X, objective_fn, constraint, ...)` keeps the reference's signature and return value
`(X, SolveStats)`.  When `objective_fn` is the bound `MDE.average_distortion` of a problem whose
distortion function and constraint the CUDA path supports, the whole solve -- L-BFGS history,
strong-Wolfe line search, projections, statistics -- runs device-resident through
`mde_solver_*` (include/mde_b200.h); X is updated in place and returned.  A distortion function that is
an arbitrary callable runs on the same solver, its torch code inside every step (pymde_b200/external.py)."""
import ctypes as C
import time

import numpy as np
import torch

from . import _lib
from . import constraints
from . import util


class SolveStats(object):
    """Summary statistics for a solve (fields of pymde/optim.py:30-47)."""

    def __init__(self, average_distortions, residual_norms, step_size_percents, solve_time, times,
                 snapshots, snapshot_every):
        self.average_distortions = average_distortions
        self.residual_norms = residual_norms
        self.step_size_percents = step_size_percents
        self.solve_time = solve_time
        self.iterations = len(average_distortions)
        self.times = times
        self.snapshots = snapshots
        self.snapshot_every = snapshot_every
        self.func_evals = None  # closure evaluations (extension: the reference does not report it)

    def __str__(self):
        return ("SolveStats:\n\taverage distortion {0:.3g}\n\tresidual norm {1:.3g}\n"
                "\tsolve_time (s) {2:.3g}\n\titerations {3}".format(
                    self.average_distortions[-1], self.residual_norms[-1], self.solve_time, self.iterations))

    def _repr_pretty_(self, p, cycle):
        del cycle
        p.text(self.__str__())


class DeviceSolver(object):
    """Owner of one `mde_solver_t`."""

    def __init__(self, layout, n, m, constraint, memory_size, max_iter, world_size=1, allreduce=None,
                 exchange=None, rank=0, external=None, constraint_part=None):
        lib = _lib.load()
        self.lib = lib
        self.layout = layout  # keep the edge layout alive
        self.device = layout.device
        self.n, self.m = int(n), int(m)
        opts = _lib.mde_solver_opts_t()
        opts.constraint = _lib.CONSTRAINT_CUSTOM if constraint_part is not None else int(constraint._solver_id)
        opts.memory_size = int(memory_size)
        opts.max_iter = max(int(max_iter), 1)
        opts.mode = 2  # the only driver: flat CUDA graphs of gated steps
        opts.world_size = int(world_size)
        self._keep = []
        if opts.constraint == _lib.CONSTRAINT_ANCHORED:
            anchors = constraint.anchors.to(device=self.device, dtype=torch.int64).contiguous()
            values = util.as_f32_cuda(constraint.values, self.device)
            opts.n_anchors = anchors.numel()
            opts.anchors = anchors.data_ptr()
            opts.anchor_values = values.data_ptr()
            self._keep += [anchors, values]
        handle = C.c_void_p()
        self._ext = None  # pymde_b200.external.UserPart of a callable distortion function
        self._part = None  # pymde_b200.external.ConstraintPart of a user-defined constraint
        with torch.cuda.device(self.device):
            if constraint_part is not None:
                self._attach(external, constraint_part, lambda x, c: lib.mde_solver_create_custom(
                    C.byref(handle), layout.handle, self.n, self.m, C.byref(opts), x, C.byref(c),
                    util.stream_ptr(self.device)))
            elif external is None:
                _lib.check(lib.mde_solver_create(C.byref(handle), layout.handle, self.n, self.m, C.byref(opts),
                                                 util.stream_ptr(self.device)))
            else:
                self._attach(external, None, lambda x, c: lib.mde_solver_create_external(
                    C.byref(handle), layout.handle, self.n, self.m, C.byref(opts), x,
                    util.stream_ptr(self.device)))
        self.handle = handle
        self.max_iter = opts.max_iter
        self.memory_size = opts.memory_size
        self._cb = None
        self.peer_memory = False
        if int(world_size) > 1 and exchange is not None:
            # peer-memory all-reduce: export this rank's cudaIpc handle, gather everybody's, map the peers
            # (pymde_b200/dist.py::exchange_handles); the solve then runs graph-captured like on one GPU
            mine = (C.c_ubyte * _lib.IPC_HANDLE_BYTES)()
            with torch.cuda.device(self.device):
                _lib.check(lib.mde_solver_comm_export(self.handle, mine, _lib.IPC_HANDLE_BYTES))
                handles = exchange(bytes(mine))  # world_size * 64 bytes, rank order
                buf = (C.c_ubyte * len(handles)).from_buffer_copy(handles)
                _lib.check(lib.mde_solver_comm_connect(self.handle, int(rank), buf, _lib.IPC_HANDLE_BYTES,
                                                       util.stream_ptr(self.device)))
            self.peer_memory = True
        elif allreduce is not None:
            self._cb = _lib.ALLREDUCE_FN(allreduce)
            _lib.check(lib.mde_solver_set_allreduce(self.handle, self._cb, None))

    def _attach(self, ext, part, call):
        """call(descriptor of ext or None, descriptor of part or None) installs the caller's parts.  When the
        library refuses a graph (node types it cannot embed), the parts fall back to hook mode one at a time, the
        constraint's first, until it accepts them."""
        def attempt():
            return call(None if ext is None else C.byref(ext.descriptor()),
                        None if part is None else part.descriptor())
        rc = attempt()
        for p in (part, ext):
            if rc == _lib.MDE_E_UNSUPPORTED and p is not None and p.mode == "graph":
                p.use_hook()
                rc = attempt()
        _lib.check(rc)
        # after the library let go of the previous parts: their graphs and buffers may be freed now
        self._ext = ext if ext is not None else self._ext
        self._part = part if part is not None else self._part

    def set_external(self, ext):
        """Run the solves from now on with the callable's part `ext` (captured anew for every embed())."""
        with torch.cuda.device(self.device):
            self._attach(ext, None, lambda x, c: self.lib.mde_solver_set_external(self.handle, x,
                                                                                 util.stream_ptr(self.device)))

    def set_constraint_part(self, part):
        """Run the solves from now on with the user-defined constraint's part `part` (captured anew for every
        embed())."""
        with torch.cuda.device(self.device):
            self._attach(None, part, lambda x, c: self.lib.mde_solver_set_constraint_part(
                self.handle, C.byref(c), util.stream_ptr(self.device)))

    @property
    def external_mode(self):
        """"graph" or "hook" for a callable distortion function, None for a table function."""
        return None if self._ext is None else self._ext.mode

    @property
    def constraint_mode(self):
        """"graph" or "hook" for a user-defined constraint, None for a built-in one."""
        return None if self._part is None else self._part.mode

    def close(self):
        if getattr(self, "handle", None):
            self.lib.mde_solver_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def begin(self, X0, eps, max_iter=None):
        """Start a solve; `max_iter` (<= the capacity this solver was created with) caps this solve."""
        X0 = util.as_f32_cuda(X0, self.device)
        cap = self.max_iter if max_iter is None else max(1, min(int(max_iter), self.max_iter))
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mde_solver_begin_ex(self.handle, X0.data_ptr(), float(eps), cap,
                                                    util.stream_ptr(self.device)))

    def run(self, iters):
        done, conv = C.c_int(0), C.c_int(0)
        with torch.cuda.device(self.device):
            rc = self.lib.mde_solver_run(self.handle, int(iters), C.byref(done), C.byref(conv),
                                         util.stream_ptr(self.device))
        for part in (self._ext, self._part):
            if part is not None:
                part.raise_error()
        if rc == _lib.MDE_E_NAN:
            raise util.SolverError("Function or gradient evaluation returned NaN/inf.")
        _lib.check(rc)
        return done.value, bool(conv.value)

    def x_view(self):
        """Zero-copy torch view of the device iterate (valid while the solver lives)."""
        ptr = self.lib.mde_solver_x(self.handle)
        return _tensor_from_ptr(ptr, (self.n, self.m), self.device, owner=self)

    def copy_x(self, out):
        out.copy_(self.x_view())
        return out

    def stats(self, iters):
        avg = np.zeros(iters)
        res = np.zeros(iters)
        pct = np.zeros(iters)
        stp = np.zeros(iters)
        fe = C.c_int64(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mde_solver_stats(self.handle, avg.ctypes.data, res.ctypes.data, pct.ctypes.data,
                                                 stp.ctypes.data, C.byref(fe), util.stream_ptr(self.device)))
        return avg, res, pct, stp, fe.value

    def debug_lbfgs(self):
        """L-BFGS state of a solve paused between two run() calls (diagnostics): a dict of CPU tensors g, g_prev, d
        (n, m), S, Y (count, n, m) in logical order, oldest first, and the numbers count, H_diag, n_iter."""
        nm = self.n * self.m
        vec = [torch.empty(nm, dtype=torch.float32) for _ in range(3)]
        S = torch.empty((self.memory_size, nm), dtype=torch.float32)
        Y = torch.empty_like(S)
        count, h_diag, n_iter = C.c_int(0), C.c_double(0.0), C.c_int(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.mde_solver_debug_lbfgs(self.handle, *[t.data_ptr() for t in vec + [S, Y]],
                                                       C.byref(count), C.byref(h_diag), C.byref(n_iter),
                                                       util.stream_ptr(self.device)))
        shape = (self.n, self.m)
        c = count.value
        return {"g": vec[0].view(shape), "g_prev": vec[1].view(shape), "d": vec[2].view(shape),
                "S": S[:c].view(c, *shape), "Y": Y[:c].view(c, *shape), "count": c, "H_diag": h_diag.value,
                "n_iter": n_iter.value}


class _PtrHolder(object):
    def __init__(self, ptr, nbytes, owner):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": (nbytes // 4,), "typestr": "<f4", "data": (ptr, False),
                                         "version": 3}


def _tensor_from_ptr(ptr, shape, device, owner):
    n = int(np.prod(shape))
    holder = _PtrHolder(ptr, n * 4, owner)
    with torch.cuda.device(device):
        t = torch.as_tensor(holder, device=device)
    return t.view(*shape)


def lbfgs(X, objective_fn, constraint, eps, max_iter, memory_size, use_line_search, use_cached_loss,
          verbose, print_every, snapshot_every, logger):
    """Projected L-BFGS (signature of pymde/optim.py:69-82).  Returns (X, SolveStats); X is
    updated in place."""
    mde = getattr(objective_fn, "__self__", None)
    fused = (mde is not None and getattr(objective_fn, "__func__", None) is type(mde).average_distortion
             and hasattr(mde, "_fused_ok") and mde._fused_ok(constraint, memory_size)
             and use_line_search and use_cached_loss)
    if not fused:
        from .generic_solver import lbfgs_generic
        return lbfgs_generic(X, objective_fn, constraint, eps, max_iter, memory_size, use_line_search,
                             use_cached_loss, verbose, print_every, snapshot_every, logger)

    start_time = time.time()
    layout = mde._layout()
    n, m = X.shape
    external = part = None
    if not mde._is_table_function():  # a callable: its torch part is captured again for every solve
        from .external import UserPart
        external = UserPart(mde.distortion_function, layout.p, layout.device)
    if not constraints.is_builtin(constraint):  # a user-defined constraint: the same, for its two projections
        from .external import ConstraintPart
        part = ConstraintPart(constraint, X)
    solver = mde._solver(constraint, memory_size, max_iter, external, part)
    solver.begin(X, eps, max_iter)
    snapshots, times = [], []
    digits = len(str(max_iter))
    need_host_steps = verbose or snapshot_every is not None
    done, converged = 0, False
    start = time.time()
    if max_iter > 0:
        if not need_host_steps:
            done, converged = solver.run(max_iter)
            times = [time.time() - start] * done
        else:
            # keep the reference's per-iteration logging / snapshot cadence
            while done < max_iter and not converged:
                if snapshot_every is not None and done % snapshot_every == 0:
                    snapshots.append(solver.x_view().detach().cpu().clone())
                prev = done
                done, converged = solver.run(1)
                times.append(time.time() - start)
                if done == prev:
                    break
                if verbose and ((prev % print_every == 0) or (prev == max_iter - 1)):
                    avg, res, pct, stp, _ = solver.stats(done)
                    logger.info("iteration %0*d | distortion %6f | residual norm %g | step length %g | "
                                "percent change %g" % (digits, prev, avg[-1], res[-1], stp[-1], pct[-1]))
            if verbose and converged:
                avg, res, pct, stp, _ = solver.stats(done)
                logger.info("Converged in %03d iterations, with residual norm %g" % (done, res[-1]))
    avg, res, pct, stp, fe = solver.stats(done)
    solver.copy_x(X)
    torch.cuda.current_stream(X.device).synchronize()
    tot_time = time.time() - start_time
    stats = SolveStats(list(avg), list(res), list(pct), tot_time, times, snapshots, snapshot_every)
    stats.func_evals = fe
    stats.step_lengths = list(stp)
    return X, stats
