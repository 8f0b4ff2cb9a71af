"""Distortion functions that are arbitrary Python callables, and user-defined constraints, on the device-resident
solver.

The reference accepts any callable mapping the (p,) distances to (p,) distortions with torch ops
(pymde/problem.py:36-193).  Inside a solver step the library computes the distances d, the callable's
torch code computes what `_ExternalAverageDistortion.forward` computes,

    fpp  = d mean(f(d)) / d d    (fp32, by autograd)
    loss = f(d).sum() in fp64,

and the library's kernels turn fpp into the gradient (include/mde_b200.h, `mde_external_t`).  The torch part
runs in one of two modes:

  graph  (default) captured as a CUDA graph once per `embed()`; the library adds it as a child node to every
         step of its own step graphs.  Tensors the callable reads are read when the graph runs, so in-place
         changes to them are seen; a rebound attribute is seen from the next `embed()` on.
  hook   the library calls back into Python at every evaluation and the torch ops are enqueued on the solver's
         stream.  Used when the callable synchronises with the host (boolean-mask indexing, `.item()`), when it
         draws random numbers (a captured draw would repeat at every replay: nothing advances the generator
         outside `CUDAGraph.replay()`), when the capture fails, or when the library refuses the graph.

PYMDE_B200_EXTERNAL=graph|hook forces a mode (graph raises if the callable cannot be captured),
PYMDE_B200_EXTERNAL=generic sends such problems to the host-stepped solver (generic_solver.py).

A user-defined constraint (any `Constraint` subclass, pymde/constraints.py:7-91) runs on the device solver only
when asked for, PYMDE_B200_CONSTRAINT=device|graph|hook (unset or `generic`: the host-stepped solver).  Its two
methods run on staging buffers the library fills and reads back with gated copies (include/mde_b200.h,
`mde_constraint_part_t`): `project_onto_constraint(U)` after the iterate moved, `project_onto_tangent_space(Xt, Gt)`
after every evaluation, in the same two modes (`device`: graph, hook where it cannot be captured)."""
import os
import warnings

import torch

from . import _lib

_MODES = ("graph", "hook", "generic")
_CONSTRAINT_MODES = ("device", "graph", "hook", "generic")


def forced_mode():
    """The mode PYMDE_B200_EXTERNAL asks for, or None."""
    v = os.environ.get("PYMDE_B200_EXTERNAL", "")
    if v and v not in _MODES:
        raise ValueError("PYMDE_B200_EXTERNAL must be one of %s, got %r" % ("|".join(_MODES), v))
    return v or None


def constraint_mode():
    """The path PYMDE_B200_CONSTRAINT asks for user-defined constraints: "device", "graph" or "hook", or None for
    the host-stepped solver (unset or "generic")."""
    v = os.environ.get("PYMDE_B200_CONSTRAINT", "")
    if v and v not in _CONSTRAINT_MODES:
        raise ValueError("PYMDE_B200_CONSTRAINT must be one of %s, got %r" % ("|".join(_CONSTRAINT_MODES), v))
    return None if v in ("", "generic") else v


def capture(device, runs, what, forced, var):
    """Capture each of the callables `runs` (torch ops, no arguments) into a CUDA graph of its own and return the
    graphs, or None when they have to run as host hooks: `what` synchronises with the host, draws random numbers, or
    its capture fails.  Two warm-up rounds run first on a side stream (lazy initialisation stays out of the graphs);
    a host synchronisation raises there under torch's sync debug mode.  `forced` == "graph" raises ValueError instead
    of returning None."""
    why = None
    side = torch.cuda.Stream(device)
    side.wait_stream(torch.cuda.current_stream(device))
    index = device.index if device.index is not None else torch.cuda.current_device()
    gen = torch.cuda.default_generators[index]
    offset = gen.get_offset()
    with torch.cuda.device(device), torch.cuda.stream(side):
        prev = torch.cuda.get_sync_debug_mode()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for _ in range(2):
                for run in runs:
                    run()
        except RuntimeError as exc:
            if "synchronizing" not in str(exc):
                raise
            why = "%s synchronises with the host" % what
        finally:
            torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.current_stream(device).wait_stream(side)
    if why is None and gen.get_offset() != offset:
        why = "%s draws random numbers" % what
    graphs = []
    for run in runs if why is None else ():
        graph = torch.cuda.CUDAGraph(keep_graph=True)
        try:
            with warnings.catch_warnings(), torch.cuda.graph(graph, stream=side):
                # an empty graph is legitimate here (a tangent projection that returns Z as it is)
                warnings.filterwarnings("ignore", message="The CUDA Graph is empty")
                run()
        except Exception as exc:  # noqa: BLE001 -- any capture failure leaves the part to hook mode
            why = "its capture failed (%s)" % (exc,)
            break
        graphs.append(graph)
    if why is None:
        return graphs
    if forced == "graph":
        raise ValueError("%s=graph, but %s" % (var, why))
    return None


class _Part(object):
    """What the two kinds of caller's parts share: the mode, the hook's stream lookup and its error."""
    _var = None

    def __init__(self, device):
        self.device = torch.device(device)
        self.error = None  # an exception raised in hook mode, re-raised after the solver returns
        self._cb = None
        self._streams = {}

    def _stream(self, stream):
        s = self._streams.get(stream)
        if s is None:  # (ctypes passes the legacy default stream, 0, as None)
            cur = torch.cuda.current_stream(self.device)
            s = cur if (stream or 0) == cur.cuda_stream else torch.cuda.ExternalStream(stream, device=self.device)
            self._streams[stream] = s
        return s

    def _call(self, stream, fn):
        try:
            with torch.cuda.stream(self._stream(stream)):
                fn()
            return 0
        except BaseException as exc:  # never let an exception cross the C boundary (as dist.make_allreduce)
            self.error = exc
            return _lib.MDE_E_INVALID

    def use_hook(self):
        """Fall back to hook mode (the library refused the captured graph)."""
        if self.forced == "graph":
            raise ValueError("%s=graph, but the captured graph holds nodes the solver cannot embed" % self._var)
        self.graphs = None
        self.mode = "hook"

    def raise_error(self):
        if self.error is not None:
            exc, self.error = self.error, None
            raise exc


class UserPart(_Part):
    """The callable's share of one evaluation, on static buffers the solver reads and writes: `d` (p,) fp32,
    `fpp` (p,) fp32 and `loss` (1,) fp64.  Kept alive with the solver (the captured graph points into them)."""
    _var = "PYMDE_B200_EXTERNAL"

    def __init__(self, f, p, device):
        super(UserPart, self).__init__(device)
        self.f = f
        self.d = torch.ones(int(p), dtype=torch.float32, device=self.device)
        self.fpp = torch.zeros(int(p), dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.graphs = None
        self.forced = forced_mode()
        if self.forced != "hook":
            self.graphs = capture(self.device, [self.run], "the callable", self.forced, self._var)
        self.mode = "hook" if self.graphs is None else "graph"

    @property
    def graph(self):
        return None if self.graphs is None else self.graphs[0]

    def run(self):
        """fpp and loss from the current d (the body of _ExternalAverageDistortion.forward)."""
        d = self.d.detach().requires_grad_(True)
        with torch.enable_grad():
            fd = self.f(d)
            (fpp,) = torch.autograd.grad(fd.mean(), d)
        self.fpp.copy_(fpp)
        self.loss.copy_(fd.detach().sum(dtype=torch.float64).reshape(1))

    def descriptor(self):
        x = _lib.mde_external_t()
        x.d, x.fpp, x.loss = self.d.data_ptr(), self.fpp.data_ptr(), self.loss.data_ptr()
        if self.mode == "graph":
            x.graph = self.graph.raw_cuda_graph()
        else:
            self._cb = _lib.EXTERNAL_FN(self._hook)
            x.fn = self._cb
        return x

    def _hook(self, user, d, fpp, loss, stream):
        return self._call(stream, self.run)


class ConstraintPart(_Part):
    """A user-defined constraint's share of every step, on staging buffers of npad fp32 each (the solver's padded
    vector length) with (n, m) views: `U` holds the iterate to retract, `Xt` and `Gt` the iterate and the gradient to
    project onto the tangent space.  The methods are called with inplace=True under torch.no_grad(); a method that
    returns another tensor has it copied into the staging buffer (as the host-stepped solver uses the return value).
    The buffers start as X0 (and a zero gradient), so the warm-up runs on a meaningful iterate.  Kept alive with the
    solver (the captured graphs point into the buffers)."""
    _var = "PYMDE_B200_CONSTRAINT"

    def __init__(self, constraint, X0):
        super(ConstraintPart, self).__init__(X0.device)
        n, m = X0.shape
        npad = (n * m + 31) // 32 * 32
        self.constraint = constraint
        self.u, self.xt, self.gt = (torch.zeros(npad, dtype=torch.float32, device=self.device) for _ in range(3))
        self.U, self.Xt, self.Gt = (b[: n * m].view(n, m) for b in (self.u, self.xt, self.gt))
        self.U.copy_(X0)
        self.Xt.copy_(X0)
        self.graphs = None
        self.forced = constraint_mode()
        if self.forced != "hook":
            self.graphs = capture(self.device, [self.retract, self.tangent], "the constraint", self.forced, self._var)
        self.mode = "hook" if self.graphs is None else "graph"

    def retract(self):
        with torch.no_grad():
            out = self.constraint.project_onto_constraint(self.U, inplace=True)
            if out is not self.U:
                self.U.copy_(out)

    def tangent(self):
        with torch.no_grad():
            out = self.constraint.project_onto_tangent_space(self.Xt, self.Gt, inplace=True)
            if out is not self.Gt:
                self.Gt.copy_(out)

    def descriptor(self):
        c = _lib.mde_constraint_part_t()
        c.u, c.xt, c.gt = self.u.data_ptr(), self.xt.data_ptr(), self.gt.data_ptr()
        if self.mode == "graph":
            c.retract_graph, c.tangent_graph = (g.raw_cuda_graph() for g in self.graphs)
        else:
            self._cb = _lib.CONSTRAINT_FN(self._hook)
            c.fn = self._cb
        return c

    def _hook(self, user, which, stream):
        return self._call(stream, self.retract if which == 0 else self.tangent)
