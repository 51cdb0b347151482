"""Record the lower problem's forward as an aten-level op tape.

The drop-in boundary hands the engine an opaque Python closure (``curr.training_step_exec``), not a
layer list (SURVEY.md §7 hard part 1).  To run the Hessian-vector products with hand-written kernels
the engine needs the structure, so the prologue's forward -- which the reference also runs once per
call (neumann.py:31, cg.py:27) -- is executed under a ``TorchDispatchMode`` that logs every aten op
with its actual input/output tensors.  PyTorch still executes the forward itself (it goes through
user code and the upper module); ``lower.py`` then turns the tape into the second-order plan.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Any, Callable, List, Sequence, Tuple

import torch
from torch.utils._python_dispatch import TorchDispatchMode


_NAMES: dict = {}   # OpOverload -> "aten.addmm.default" (str() of an overload costs ~3 us; asked ~1.3 times per op)


@dataclass
class TapeOp:
    func: Any           # torch._ops.OpOverload
    args: tuple
    kwargs: dict
    out: Any            # Tensor | tuple | list

    @property
    def name(self) -> str:
        n = _NAMES.get(self.func)
        if n is None:
            n = _NAMES[self.func] = str(self.func)  # e.g. "aten.addmm.default"
        return n


@dataclass
class Tape:
    ops: List[TapeOp] = field(default_factory=list)
    params: List[torch.Tensor] = field(default_factory=list)
    loss: torch.Tensor = None


# ---- native prologue pieces (SURVEY.md 8 f2) ------------------------------------------------------------------------
# Training-mode BatchNorm forward on a large channels-first CUDA activation: PyTorch launches one block per channel;
# csrc/bn_fwd.cu spreads each channel over many blocks and makes the prologue shorter.  OPT-IN (BB200_PROLOGUE_BN_MIN=<numel>), off by
# default: its statistics differ from aten's in the last fp32 bits, 7e-5 of the bf16 outputs round the other way, and
# a bf16 4-conv net amplifies that (max-pool / ReLU switches, small-batch statistics) to a 2e-2 ... 6e-2 change of
# the hypergradient -- inside the reference's own bf16-vs-fp64 gap, but outside the 1e-2 engine-vs-reference bar,
# which only holds while both sides differentiate bit-identical base activations.  So by default every op of the
# lower forward runs on PyTorch, exactly as in the reference (neumann.py:31, cg.py:27).
_BN_FWD_OPS = {"aten.native_batch_norm.default": True, "aten._native_batch_norm_legit.default": True,
               "aten._native_batch_norm_legit.no_stats": False}   # name -> has running statistics arguments
native_bn_min_numel = int(os.environ.get("BB200_PROLOGUE_BN_MIN", "0"))   # <= 0: off (default)
native_bn_calls = 0


def _native_bn_forward(name, args, kwargs):
    """(out, save_mean, save_invstd) of a training-mode batch norm computed by bb_bn_forward, or None when this call
    is left to PyTorch (small / CPU / eval mode / exotic layouts)."""
    global native_bn_calls
    if kwargs or native_bn_min_numel <= 0:
        return None
    if _BN_FWD_OPS[name]:
        if len(args) != 8:
            return None
        x, w, b, rm, rv, training, momentum, eps = args
    else:
        if len(args) != 6:
            return None
        x, w, b, training, momentum, eps = args
        rm = rv = None
    if not (training and isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == 4 and x.is_contiguous()
            and x.dtype in (torch.float32, torch.bfloat16) and x.numel() >= native_bn_min_numel
            and x.shape[1] <= 65535 and x.numel() // x.shape[1] > 1):
        return None
    for t in (w, b, rm, rv):
        if t is not None and not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            return None
    from . import _native as N

    n, c, hw = x.shape[0], x.shape[1], x.shape[2] * x.shape[3]
    with torch.cuda.device(x.device):
        y = torch.empty_like(x)
        stats = torch.empty((3, c), dtype=torch.float32, device=x.device)
        splits = N.lib().bb_bn_forward_splits(n, c)
        ws = torch.empty(2 * c * splits, dtype=torch.float64, device=x.device)
        N.call("bb_bn_forward", x.data_ptr(), 0 if x.dtype == torch.float32 else 1,
               w.data_ptr() if w is not None else None, b.data_ptr() if b is not None else None, float(eps),
               y.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(), ws.data_ptr(), n, c, hw,
               torch.cuda.current_stream().cuda_stream)
        if rm is not None:      # running statistics exactly as aten does: (1 - momentum) * running + momentum * batch
            rm.mul_(1.0 - momentum).add_(stats[0], alpha=momentum)
        if rv is not None:
            rv.mul_(1.0 - momentum).add_(stats[2], alpha=momentum)
    native_bn_calls += 1
    return y, stats[0], stats[1]


class _Recorder(TorchDispatchMode):
    def __init__(self, tape: Tape):
        super().__init__()
        self.tape = tape

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = None
        name = _NAMES.get(func)
        if name is None:
            name = _NAMES[func] = str(func)
        if name in _BN_FWD_OPS:
            out = _native_bn_forward(name, args, kwargs)
        if out is None:
            out = func(*args, **kwargs)
        # keeping args/out alive keeps id() stable and the base activations resident for the K-loop
        self.tape.ops.append(TapeOp(func, args, kwargs, out))
        return out


def record_tape(fn: Callable[[], Any], params: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, Tape]:
    """Run ``fn`` (the lower ``training_step_exec``) and return ``(loss, tape)``.  The autograd graph
    above the dispatch layer is built as usual, so the caller can still differentiate the loss."""
    tape = Tape(params=list(params))
    with _Recorder(tape):
        out = fn()
    loss = out["loss"] if isinstance(out, dict) else (out[0] if isinstance(out, (tuple, list)) else out)
    tape.loss = loss
    return loss, tape


# --------------------------------------------------------------------------------------------------------------------
# tape signatures (plan cache, engine.py): two tapes with equal signatures are the same computation on different values
# --------------------------------------------------------------------------------------------------------------------
def op_tensors(op: TapeOp) -> List[torch.Tensor]:
    """Every tensor an op touches, in a fixed order (args, kwargs by key, outputs; nested lists flattened).  The
    position in this list identifies "the same tensor" across two tapes of equal signature."""
    out: List[torch.Tensor] = []

    def walk(x):
        if isinstance(x, torch.Tensor):
            out.append(x)
        elif isinstance(x, (list, tuple)):
            for y in x:
                walk(y)

    walk(op.args)
    if op.kwargs:
        for k in sorted(op.kwargs):
            walk(op.kwargs[k])
    walk(op.out)
    return out


def _plain(x):
    if isinstance(x, torch.Tensor):
        return None
    if isinstance(x, (list, tuple)):
        return tuple(_plain(y) for y in x)
    if isinstance(x, (int, float, bool, str, type(None), torch.dtype, torch.device, torch.layout, torch.memory_format)):
        return x
    return repr(x)


def tape_signature(tape: Tape, extra=()) -> tuple:
    """Hashable description of the recorded computation: op sequence, non-tensor arguments, and for every tensor slot
    either (shape, stride, dtype, requires_grad) at its first appearance or the index of that first appearance
    (the dataflow).  Parameter storage addresses are part of it: a cached plan points at them."""
    seen: dict = {}
    parts = [tuple(extra), tuple((p.data_ptr(), tuple(p.shape), p.dtype) for p in tape.params)]
    for p in tape.params:
        seen[id(p)] = len(seen)
    for op in tape.ops:
        items = [op.func, _plain(op.args), _plain(tuple(sorted(op.kwargs.items()))) if op.kwargs else None]
        for t in op_tensors(op):
            j = seen.get(id(t))
            if j is None:
                seen[id(t)] = len(seen)
                items.append((tuple(t.shape), t.stride(), t.dtype, t.requires_grad, t.device.index))
            else:
                items.append(j)
        parts.append(tuple(items))
    loss = tape.loss
    parts.append(seen.get(id(loss), -1))
    return tuple(parts)


def tensor_locator(tape: Tape) -> dict:
    """id(tensor) -> (op index, position in op_tensors) of its first appearance."""
    loc: dict = {}
    for i, op in enumerate(tape.ops):
        for k, t in enumerate(op_tensors(op)):
            if id(t) not in loc:
                loc[id(t)] = (i, k)
    return loc
