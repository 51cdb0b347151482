"""Call-level orchestration shared by the neumann / cg plugins.

One hypergradient call =
  prologue   lower forward on ``curr.cur_batch``, recorded as an aten op tape   (reference neumann.py:31, cg.py:27;
             the reference's ``grad(..., create_graph=True)`` at :34 / :30 is NOT needed by the native path)
  K-loop     K Hessian-vector products + vector updates      (reference neumann.py:59-66, cg.py:34-56)
             -> CUDA: the native second-order tape (csrc/plan.cu, K5-K9) + flat-arena kernels K1-K3
                (csrc/kloop.cu), one CUDA graph per iteration
  epilogue   ``-(d^2 L_in/d lambda d w)^T x``                 (reference neumann.py:44-54, cg.py:58-68)
             -> one more tangent forward/backward along x gives d(g.x)/dB for every upper-dependent tensor B of
                the lower forward; a first-order ``autograd`` backward through the (small) upper graph finishes.
                Graphs whose upper dependence the lowering cannot capture fall back to the reference's double
                backward for this step only.
(development mode ``hvp="autograd"``: H.v by torch's double backward around the same K1-K3 kernels)

There is no CPU path: everything here raises without a CUDA device.
"""
from __future__ import annotations

import os
import warnings
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import torch

from . import _native as N
from .arena import ArenaLayout, pack, stream_ptr


@dataclass
class Settings:
    # "native": hand-written second-order tape; "autograd" (development only): torch double backward
    hvp: str = os.environ.get("BB200_HVP", "native")
    cuda_graph: bool = True   # capture one K-loop iteration and replay it
    # mixed second derivative from the tape's boundary adjoint-tangents (one extra pass) instead of autograd's
    # double backward; automatically off for graphs whose upper dependence the lowering could not capture
    native_epilogue: bool = os.environ.get("BB200_EPILOGUE", "native") == "native"
    record_events: bool = True


settings = Settings()


@dataclass
class CallStats:
    """Filled by every call; bench.py reads the CUDA events after a synchronize."""
    method: str = ""
    iterations: int = 0
    n_params: int = 0
    ev_start: Optional[torch.cuda.Event] = None
    ev_end: Optional[torch.cuda.Event] = None
    plan_launches_per_iter: int = 0
    extra: dict = field(default_factory=dict)

    def kloop_ms(self) -> float:
        self.ev_end.synchronize()
        return self.ev_start.elapsed_time(self.ev_end)


last_stats = CallStats()


class Workspace:
    """Zero-initialised device block for the K-loop scalars / reduction slots (bb_kloop_scalars)."""

    _cache = {}

    def __init__(self, device):
        nbytes = N.lib().bb_kloop_ws_bytes()
        self.buf = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        self.scalars = self.buf[:64].view(torch.float64)  # rr, php, rr_new, alpha, beta, sumsq, eps, inv_2eps

    @property
    def ptr(self):
        return self.buf.data_ptr()

    def scalar_ptr(self, idx: int) -> int:
        return self.buf.data_ptr() + 8 * idx

    @classmethod
    def get(cls, device) -> "Workspace":
        key = (device.type, device.index)
        ws = cls._cache.get(key)
        if ws is None:
            ws = cls._cache[key] = cls(device)
        return ws


def lower_gradient(curr):
    """Reference prologue (neumann.py:31-36, cg.py:27-32): lower loss on the last batch and its gradient with a
    graph.  Only the development mode ``hvp="autograd"`` and the autograd-epilogue fallback need it."""
    params = curr.trainable_parameters()
    in_loss = curr.training_step_exec(curr.cur_batch)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        in_grad = torch.autograd.grad(in_loss, params, create_graph=True)
    return in_loss, in_grad


class AutogradHvp:
    """Development mode: H.d by torch double backward, result packed into the hv arena."""

    def __init__(self, in_grad, params, layout: ArenaLayout, d_arena: torch.Tensor, hv_arena: torch.Tensor):
        self.in_grad, self.params, self.layout = in_grad, params, layout
        self.d_views = layout.views(d_arena)
        self.hv_arena = hv_arena
        self.launches_per_iter = 1

    def __call__(self):
        hv = torch.autograd.grad(self.in_grad, self.params, grad_outputs=self.d_views, retain_graph=True)
        pack(self.layout, hv, self.hv_arena)


class _nvtx:
    """NVTX range around a call phase (visible in nsys / ncu timelines; free when no profiler is attached)."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        torch.cuda.nvtx.range_pop()


def _events():
    if not settings.record_events:
        return None, None
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


class _PlanEntry:
    """What one traced computation needs on the device: the native plan and the K-loop arenas its descriptors and
    captured graphs point into."""

    def __init__(self, plan, layout, d, hd, acc, out):
        self.plan, self.layout, self.d, self.hd, self.acc, self.out = plan, layout, d, hd, acc, out
        self.r = None
        self.in_use = False


class PlanCache:
    """Plans keyed by tape signature (trace.tape_signature).  A training loop calls the plugin every few steps with
    the same model and batch shape: tracing the forward is unavoidable (the reference runs it too, neumann.py:31),
    but lowering, descriptor building, buffer allocation, tensor-map encoding and CUDA-graph capture are paid once --
    a hit copies the new forward's values behind the pointers the plan already holds (HvpPlan.rebind)."""

    def __init__(self):
        import collections

        self.entries = collections.OrderedDict()
        self.hits = self.misses = 0

    @property
    def capacity(self) -> int:
        return int(os.environ.get("BB200_PLAN_CACHE", "4"))

    def get(self, key):
        e = self.entries.get(key)
        if e is not None and not e.in_use:
            self.entries.move_to_end(key)
            return e
        return None

    def put(self, key, entry):
        if self.capacity <= 0:
            return
        self.entries[key] = entry
        self.entries.move_to_end(key)
        while len(self.entries) > self.capacity:
            k, old = next(iter(self.entries.items()))
            if old.in_use and len(self.entries) <= self.capacity + 2:
                break
            del self.entries[k]

    def clear(self):
        self.entries.clear()


plan_cache = PlanCache()


class HypergradientCall:
    """One ``fn(vector, curr, prev, sync)`` invocation split into its three phases so that
    ``bench.py`` can time the K-loop alone: ``__init__`` = prologue (+ arenas, + native plan),
    ``solve`` = K-loop, ``finish`` = epilogue."""

    def __init__(self, curr, method: str):
        N.require_cuda()
        self.curr, self.method = curr, method
        cfg = curr.config
        if method == "neumann":
            self.K, self.alpha = int(cfg.neumann_iterations), float(cfg.neumann_alpha)
        elif method == "cg":
            self.K, self.alpha = int(cfg.cg_iterations), float(cfg.cg_alpha)
        else:
            raise ValueError(method)
        params = curr.trainable_parameters()
        self.dev = params[0].device
        self.entry = None
        self.in_grad = None
        with torch.cuda.device(self.dev):
            self.ws = Workspace.get(self.dev)
            if settings.hvp == "native":
                self._init_native(curr, params)
            else:
                lay = self.layout = ArenaLayout.like(params)
                # d = direction the HVP is taken along (v for Neumann, p for CG); hd = H.d
                self.d, self.hd, self.acc, self.out = (lay.new(self.dev) for _ in range(4))
                self.in_loss, self.in_grad = lower_gradient(curr)
                self.tape = None
                self.hvp = AutogradHvp(self.in_grad, params, lay, self.d, self.hd)
                self.native_epilogue = False
            self.r = None
            if method == "cg":
                if self.entry is not None:
                    if self.entry.r is None:
                        self.entry.r = self.layout.new(self.dev)
                    self.r = self.entry.r
                else:
                    self.r = self.layout.new(self.dev)

    def _init_native(self, curr, params):
        # prologue = the lower forward only (reference neumann.py:31 / cg.py:27), recorded as a tape; the
        # gradient-with-graph of neumann.py:34 is needed only if the epilogue has to fall back to autograd
        from .plan import HvpPlan
        from .trace import record_tape, tape_signature

        with _nvtx("betty_b200:prologue:trace"):
            self.in_loss, tape = record_tape(lambda: curr.training_step_exec(curr.cur_batch), params)
        entry = None
        key = None
        if plan_cache.capacity > 0:
            with _nvtx("betty_b200:prologue:signature"):
                key = tape_signature(tape, extra=(bool(settings.cuda_graph), self.dev.index))
            entry = plan_cache.get(key)
        if entry is not None:
            with _nvtx("betty_b200:prologue:rebind"):
                if not entry.plan.rebind(tape):
                    plan_cache.entries.pop(key, None)   # do not keep the stale plan alive next to its replacement
                    entry = None
        if entry is not None:
            plan_cache.hits += 1
            self.tape = entry.plan.tape
        else:
            plan_cache.misses += key is not None
            lay = ArenaLayout.like(params)
            d, hd, acc, out = (lay.new(self.dev) for _ in range(4))
            with _nvtx("betty_b200:prologue:plan"):
                plan = HvpPlan(tape, params, lay, d, hd)
            entry = _PlanEntry(plan, lay, d, hd, acc, out)
            if key is not None:
                plan_cache.put(key, entry)
            self.tape = tape
        entry.in_use = True
        self.entry = entry
        self.hvp, self.layout = entry.plan, entry.layout
        self.d, self.hd, self.acc, self.out = entry.d, entry.hd, entry.acc, entry.out
        self.native_epilogue = settings.native_epilogue and self.hvp.g.native_epilogue_ok

    def release(self):
        """Hand the cached plan back (end of the call)."""
        if self.entry is not None:
            self.entry.in_use = False
            self.entry = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def solve(self, vector: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        with torch.cuda.device(self.dev):
            return self._solve(vector)

    def _solve(self, vector: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        global last_stats
        lay, s, n = self.layout, stream_ptr(), self.layout.total
        K, alpha, hvp = self.K, self.alpha, self.hvp
        d, hd, acc = self.d, self.hd, self.acc
        torch.cuda.nvtx.range_push(f"betty_b200:kloop:{self.method}:K={K}")
        pack(lay, vector, d)
        e0, e1 = _events()
        if self.method == "neumann":
            # reference neumann.py:59-66:  v <- v - alpha H v ; p <- p + v ; return alpha p
            acc.copy_(d)
            if e0 is not None:
                e0.record()
            if hasattr(hvp, "neumann_loop"):
                hvp.neumann_loop(K, alpha, d, acc, hd)
            else:
                for _ in range(K):
                    hvp()
                    N.call("bb_neumann_update", d.data_ptr(), acc.data_ptr(), hd.data_ptr(), alpha, 0.0, n, s)
            if e1 is not None:
                e1.record()
            N.call("bb_scale", self.out.data_ptr(), acc.data_ptr(), alpha, n, s)
        else:
            # reference cg.py:34-56 with x = acc, p = d
            r, ws = self.r, self.ws
            r.copy_(d)
            acc.zero_()
            if e0 is not None:
                e0.record()
            if hasattr(hvp, "cg_loop"):
                hvp.cg_loop(K, alpha, acc, r, d, hd, ws)
            else:
                for k in range(K):
                    hvp()
                    N.call("bb_cg_dots", r.data_ptr(), hd.data_ptr(), d.data_ptr(), alpha, 0.0, int(k == 0), n, ws.ptr, s)
                    N.call("bb_cg_update_xr", acc.data_ptr(), r.data_ptr(), d.data_ptr(), hd.data_ptr(), 0.0, n, ws.ptr, s)
                    N.call("bb_cg_update_p", d.data_ptr(), r.data_ptr(), n, ws.ptr, s)
            if e1 is not None:
                e1.record()
            N.call("bb_scale", self.out.data_ptr(), acc.data_ptr(), alpha, n, s)
        torch.cuda.nvtx.range_pop()
        last_stats = CallStats(self.method, K, lay.n_logical, e0, e1, getattr(hvp, "launches_per_iter", 0))
        return lay.views(self.out)

    def finish(self, prev, x, sync):
        try:
            with torch.cuda.device(self.dev):
                if self.native_epilogue:
                    with _nvtx("betty_b200:epilogue:native"):
                        return chain_boundary_seeds(self.hvp.mixed_seeds(self.out), prev, sync)
                if self.in_grad is None:
                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")
                        self.in_grad = torch.autograd.grad(self.in_loss, self.curr.trainable_parameters(),
                                                           create_graph=True)
                return mixed_product(self.in_grad, prev, x, sync)
        finally:
            self.release()


def chain_boundary_seeds(seeds, prev, sync: bool):
    """Finish the native epilogue: ``seeds`` = [(B, d(g.x)/dB)] for every upper-dependent tensor B that enters
    the lower forward.  -(d^2 L_in/d lambda d w)^T x = -sum_B (dB/d lambda)^T seed_B, one ordinary first-order
    backward through the (small) upper graph.  ``sync`` goes through ``torch.autograd.backward`` so the upper
    module's DDP reducer all-reduces it, as in the reference (neumann.py:44-49, cg.py:58-63)."""
    lam = prev.trainable_parameters()
    outs = [b for b, _ in seeds]
    grads = [-(g.to(b.dtype)) for b, g in seeds]
    if sync:
        if outs:
            torch.autograd.backward(outs, grad_tensors=grads, inputs=lam)
        return None
    if not outs:
        return [torch.zeros_like(p) for p in lam]
    res = torch.autograd.grad(outs, lam, grad_outputs=grads, allow_unused=True)
    return [torch.zeros_like(p) if r is None else r for r, p in zip(res, lam)]


def mixed_product(in_grad, prev, x: Sequence[torch.Tensor], sync: bool):
    """Epilogue: -(d^2 L_in / d lambda d w)^T x.  ``sync`` accumulates into ``.grad`` through
    ``torch.autograd.backward`` so the upper module's DDP reducer averages it across ranks
    (reference neumann.py:44-54, cg.py:58-68)."""
    lam = prev.trainable_parameters()
    if sync:
        torch.autograd.backward(in_grad, inputs=lam, grad_tensors=[-xi for xi in x])
        return None
    out = torch.autograd.grad(in_grad, lam, grad_outputs=list(x))
    return [-g for g in out]
