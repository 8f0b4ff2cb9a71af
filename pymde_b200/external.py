"""Distortion functions that are arbitrary Python callables, on the device-resident solver.

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
PYMDE_B200_EXTERNAL=generic sends such problems to the host-stepped solver (generic_solver.py)."""
import os

import torch

from . import _lib

_MODES = ("graph", "hook", "generic")


def forced_mode():
    """The mode PYMDE_B200_EXTERNAL asks for, or None."""
    v = os.environ.get("PYMDE_B200_EXTERNAL", "")
    if v and v not in _MODES:
        raise ValueError("PYMDE_B200_EXTERNAL must be one of %s, got %r" % ("|".join(_MODES), v))
    return v or None


class UserPart(object):
    """The callable's share of one evaluation, on static buffers the solver reads and writes: `d` (p,) fp32,
    `fpp` (p,) fp32 and `loss` (1,) fp64.  Kept alive with the solver (the captured graph points into them)."""

    def __init__(self, f, p, device):
        self.f = f
        self.device = torch.device(device)
        self.d = torch.ones(int(p), dtype=torch.float32, device=self.device)
        self.fpp = torch.zeros(int(p), dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.graph = None
        self.error = None  # an exception raised by the callable in hook mode, re-raised after the solver returns
        self._cb = None
        self._streams = {}
        self.forced = forced_mode()
        self.mode = "hook" if self.forced == "hook" else self._capture()

    def run(self):
        """fpp and loss from the current d (the body of _ExternalAverageDistortion.forward)."""
        d = self.d.detach().requires_grad_(True)
        with torch.enable_grad():
            fd = self.f(d)
            (fpp,) = torch.autograd.grad(fd.mean(), d)
        self.fpp.copy_(fpp)
        self.loss.copy_(fd.detach().sum(dtype=torch.float64).reshape(1))

    def _capture(self):
        why = None
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        gen = torch.cuda.default_generators[index]
        offset = gen.get_offset()
        with torch.cuda.device(self.device), torch.cuda.stream(side):
            # warm-up (lazy initialisation stays out of the graph); a host synchronisation raises here
            prev = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode("error")
            try:
                for _ in range(2):
                    self.run()
            except RuntimeError as exc:
                if "synchronizing" not in str(exc):
                    raise
                why = "the callable synchronises with the host"
            finally:
                torch.cuda.set_sync_debug_mode(prev)
        torch.cuda.current_stream(self.device).wait_stream(side)
        if why is None and gen.get_offset() != offset:
            why = "the callable draws random numbers"
        if why is None:
            graph = torch.cuda.CUDAGraph(keep_graph=True)
            try:
                with torch.cuda.graph(graph, stream=side):
                    self.run()
                self.graph = graph
            except Exception as exc:  # noqa: BLE001 -- any capture failure leaves the callable to hook mode
                why = "its capture failed (%s)" % (exc,)
        if why is None:
            return "graph"
        if self.forced == "graph":
            raise ValueError("PYMDE_B200_EXTERNAL=graph, but %s" % why)
        return "hook"

    def use_hook(self):
        """Fall back to hook mode (the library refused the captured graph)."""
        if self.forced == "graph":
            raise ValueError("PYMDE_B200_EXTERNAL=graph, but the captured graph holds nodes the solver cannot embed")
        self.graph = None
        self.mode = "hook"

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
        try:
            s = self._streams.get(stream)
            if s is None:  # (ctypes passes the legacy default stream, 0, as None)
                cur = torch.cuda.current_stream(self.device)
                s = cur if (stream or 0) == cur.cuda_stream else torch.cuda.ExternalStream(stream, device=self.device)
                self._streams[stream] = s
            with torch.cuda.stream(s):
                self.run()
            return 0
        except BaseException as exc:  # never let an exception cross the C boundary (as dist.make_allreduce)
            self.error = exc
            return _lib.MDE_E_INVALID

    def raise_error(self):
        if self.error is not None:
            exc, self.error = self.error, None
            raise exc
