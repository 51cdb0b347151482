"""Second-order tape IR: the recorded aten ops lowered to a small set of nodes, each with three rules

    TF  tangent forward        t_y   = J_x(x) t_x                       (R-forward of SURVEY.md App. B)
    BB  base backward          a_x  += J_x(x)^T a_y                     (delta, once per call)
    TB  tangent backward       at_x += J^T at_y + (dJ^T/dx . t_x) a_y   (R-backward -> H.v slices)

Every lower-active value carries four same-shaped tensors: ``base`` (recorded by the forward, fp32 or
bf16 under autocast), ``t`` (tangent), ``a`` (adjoint, delta) and ``at`` (adjoint tangent); the
last three are fp32.  A parameter's ``t`` is its slice of the direction arena and its ``at`` is its
slice of the H.d arena, so the K-loop kernels read/write them with no gather/scatter.

View ops (view/transpose/select/...) create *aliases*: their buffers are the same view applied to the
parent's buffers, so they cost nothing in any pass.  Because adjoints reach a buffer through aliases
from several consumers, adjoint writes either overwrite (``beta=0``: the buffer has exactly one writer
and it covers the whole buffer) or accumulate into a buffer zeroed at the start of the pass.

The node rules are implemented twice: in CUDA (``csrc/*.cu``, the product) and in torch
(``oracle/plan_interp.py``, test infrastructure that checks this file's lowering and the rule maths on
CPU against autograd's double backward).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch


class UnsupportedGraph(NotImplementedError):
    """Raised when the lower forward contains an op the engine has no second-order rule for.
    There is deliberately no fallback (BASELINE.json north_star)."""


class Val:
    """A lower-active tensor value."""

    __slots__ = ("vid", "base", "param_index", "parent", "viewfn", "full_cover", "name", "t", "a", "at",
                 "writers", "needed", "zero_init", "ident", "boundary", "interp_only", "tfmt")

    def __init__(self, vid, base, param_index=None, parent=None, viewfn=None, full_cover=True, name="", ident=False):
        self.vid = vid
        self.base = base
        self.param_index = param_index      # index into the lower parameter list, or None
        self.parent: Optional["Val"] = parent
        self.viewfn: Optional[Callable] = viewfn
        self.full_cover = full_cover        # does this alias cover every element of its parent exactly once?
        self.name = name
        self.t = self.a = self.at = None    # root buffers, filled by the executor
        self.writers = 0                    # adjoint writers reaching this root (through aliases)
        self.needed = False
        self.zero_init = False              # root adjoint buffers must be zeroed before BB / TB
        self.ident = ident                  # alias whose buffers are *exactly* the parent's (cast, x + const)
        self.boundary = False               # upper-dependent constant (requires_grad, not from the lower params)
        self.interp_only = False            # internal value of a fused node: only the torch interpreter gives it buffers
        self.tfmt = None                    # "nhwc_bf16": t / a / at are bf16 padded NHWC [N][H+2][W+2][64], handed from
                                            # one fused block to the next as TMA operands (no fp32 NCHW buffers)

    @property
    def root(self) -> "Val":
        v = self
        while v.parent is not None:
            v = v.parent
        return v

    @property
    def is_param(self) -> bool:
        return self.root.param_index is not None and self.parent is None

    def chain_full_cover(self) -> bool:
        v, ok = self, True
        while v.parent is not None:
            ok = ok and v.full_cover
            v = v.parent
        return ok

    @property
    def shape(self):
        return tuple(self.base.shape)

    def __repr__(self):
        return f"Val#{self.vid}{tuple(self.base.shape)}{'P' if self.param_index is not None else ''}"


@dataclass
class Node:
    op: str
    ins: List[Optional[Val]]            # active inputs; None where that operand is a constant
    out: Optional[Val]
    attrs: Dict[str, Any] = field(default_factory=dict)
    beta: List[int] = field(default_factory=list)   # per input: 0 overwrite / 1 accumulate (adjoint writes)
    src: str = ""                                    # aten op it came from

    def __repr__(self):
        return f"Node({self.op}, ins={self.ins}, out={self.out})"


@dataclass
class Graph:
    nodes: List[Node]
    values: List[Val]
    params: List[Val]
    loss: Val
    stats: Dict[str, int] = field(default_factory=dict)
    boundaries: List[Val] = field(default_factory=list)   # upper-dependent tensors entering the lower tape
    native_epilogue_ok: bool = True                        # every such tensor was captured as a boundary value
    validators: List[Any] = field(default_factory=list)    # (check() -> bool, message): data-dependent refusals
    derived: List[Tuple[torch.Tensor, torch.Tensor]] = field(default_factory=list)  # (copy, source): contiguous
                                                           # copies the lowering made of strided tape views


# --------------------------------------------------------------------------------------------------
# lowering
# --------------------------------------------------------------------------------------------------
_VIEW_OPS = {
    # name -> full_cover
    "aten.view.default": True, "aten._unsafe_view.default": True, "aten.reshape.default": True,
    "aten.t.default": True, "aten.transpose.int": True, "aten.permute.default": True,
    "aten.unsqueeze.default": True, "aten.squeeze.dim": True, "aten.squeeze.default": True,
    "aten.alias.default": True, "aten.select.int": False, "aten.slice.Tensor": False,
    "aten.expand.default": True, "aten.flatten.using_ints": True,
}
_UNARY = {"aten.relu.default": "relu", "aten.gelu.default": "gelu", "aten.tanh.default": "tanh",
          "aten.sigmoid.default": "sigmoid", "aten.neg.default": "neg"}
_BN_OPS = ("aten.native_batch_norm.default", "aten._native_batch_norm_legit.default",
           "aten._native_batch_norm_legit_no_stats.default", "aten.cudnn_batch_norm.default",
           "aten._native_batch_norm_legit.no_stats", "aten._batch_norm_with_update.default",
           "aten.miopen_batch_norm.default")


def _narrow_interior(t: torch.Tensor, pads, nd: int, shape) -> torch.Tensor:
    """The un-padded interior of a constant_pad_nd output (pads are given last-dim first)."""
    for k in range(len(pads) // 2):
        dim = nd - 1 - k
        lo = pads[2 * k]
        if lo < 0 or pads[2 * k + 1] < 0:
            raise UnsupportedGraph("negative padding (cropping)")
        t = t.narrow(dim, lo, shape[dim])
    return t


def _float_outputs(out) -> List[torch.Tensor]:
    if isinstance(out, torch.Tensor):
        return [out] if out.is_floating_point() else []
    if isinstance(out, (list, tuple)):
        return [o for o in out if isinstance(o, torch.Tensor) and o.is_floating_point()]
    return []


def _is_dense(t: torch.Tensor) -> bool:
    """non-overlapping and dense: some permutation of the dims is contiguous"""
    if t.numel() <= 1:
        return True
    dims = sorted([(st, sz) for sz, st in zip(t.shape, t.stride()) if sz != 1])
    expect = 1
    for st, sz in dims:
        if st != expect:
            return False
        expect *= sz
    return True


class _Lowering:
    def __init__(self, tape):
        self.tape = tape
        self.vals: Dict[int, Val] = {}
        self.all_vals: List[Val] = []
        self.nodes: List[Node] = []
        self.params: List[Val] = []
        self.boundaries: List[Val] = []
        self.native_epilogue_ok = True
        self.validators: List[Tuple[Callable[[], bool], str]] = []   # value-dependent refusals, re-checked per call
        self.derived: List[Tuple[torch.Tensor, torch.Tensor]] = []
        self._pending_upper: set = set()
        for i, p in enumerate(tape.params):
            v = self._new(p, param_index=i, name=f"param{i}")
            self.params.append(v)

    # -- helpers ---------------------------------------------------------------------------
    def _new(self, base, **kw) -> Val:
        v = Val(len(self.all_vals), base, **kw)
        self.all_vals.append(v)
        self.vals[id(base)] = v
        return v

    def act(self, x) -> Optional[Val]:
        return self.vals.get(id(x)) if isinstance(x, torch.Tensor) else None

    def boundary(self, t: torch.Tensor) -> Optional[Val]:
        """Value for an upper-dependent constant ``t`` (requires_grad, not derived from the lower parameters).
        It takes part in every rule as an input whose tangent is identically zero; what the tangent-backward
        pass accumulates into its ``at`` buffer is d(g.x)/dt, the seed of the native epilogue
        (reference neumann.py:44-54: -(d^2 L_in / d lambda d w)^T x)."""
        if not (isinstance(t, torch.Tensor) and t.requires_grad and t.is_floating_point()):
            return None
        self._pending_upper.discard(id(t))
        v = self.vals.get(id(t))
        if v is None:
            v = self._new(t, name="boundary")
            v.boundary = True
            self.boundaries.append(v)
        return v

    def emit(self, op, ins, out_tensor, src, **attrs) -> Node:
        out = self._new(out_tensor) if out_tensor is not None else None
        n = Node(op, list(ins), out, attrs, src=src)
        self.nodes.append(n)
        return n

    def alias(self, parent: Val, out_tensor, viewfn, full_cover=True, ident=False):
        return self._new(out_tensor, parent=parent, viewfn=viewfn, full_cover=full_cover, ident=ident)

    @staticmethod
    def need_contig(v: Val, what: str):
        if not v.base.is_contiguous():
            raise UnsupportedGraph(f"{what}: needs a contiguous operand, got strides {v.base.stride()} for {v.shape}")

    # -- main loop ---------------------------------------------------------------------------
    def run(self, fold_quadratic: bool = True) -> Graph:
        for op in self.tape.ops:
            tensors = [a for a in op.args if isinstance(a, torch.Tensor)]
            for a in op.args:
                if isinstance(a, (list, tuple)):
                    tensors += [x for x in a if isinstance(x, torch.Tensor)]
            if not any(id(t) in self.vals and not self.vals[id(t)].boundary for t in tensors):
                continue  # constant w.r.t. the lower parameters (data prep, upper module forward, ...)
            outs = _float_outputs(op.out)
            if not outs:
                continue  # .item(), argmax, comparisons ...: nothing differentiable comes out (metrics, masks)
            if not any(o.requires_grad for o in outs):
                # computed under torch.no_grad() (or detached): autograd -- hence the reference -- treats the
                # result as a constant, and so must the second-order rules.  An in-place op would have kept
                # requires_grad, so the tensor object is a fresh one and nothing recorded refers to it.
                continue
            self._pending_upper = {id(t) for t in tensors
                                   if t.requires_grad and t.is_floating_point() and id(t) not in self.vals}
            n_nodes, n_vals = len(self.nodes), len(self.all_vals)
            try:
                self.lower_op(op)
            except UnsupportedGraph as e:
                # Not fatal yet: side computations (logging, accuracy) routinely use ops without a rule.  The
                # outputs become *poison* values; the call is refused only if one of them reaches the loss
                # (checked after dead-code elimination in _analyse).
                del self.nodes[n_nodes:]
                ins = [self.vals[id(t)] for t in tensors if id(t) in self.vals]
                for o in outs:
                    self.emit("poison", ins, o, op.name, error=str(e))
            if self._pending_upper and op.name not in ("aten.detach.default", "aten.detach_.default"):
                # an upper-dependent tensor entered an op in a slot this lowering treats as a plain constant:
                # the K-loop is still exact, but the mixed second derivative must then come from autograd
                self.native_epilogue_ok = False
        loss = self.vals.get(id(self.tape.loss))
        if loss is None:
            raise UnsupportedGraph("the lower loss does not depend on the lower parameters (or was produced "
                                   "outside the recorded forward)")
        if loss.base.numel() != 1:
            raise UnsupportedGraph("the lower loss must be a scalar")
        g = Graph(self.nodes, self.all_vals, self.params, loss)
        g.boundaries = self.boundaries
        g.native_epilogue_ok = self.native_epilogue_ok
        g.validators = self.validators
        g.derived = self.derived
        if fold_quadratic:
            _fold_quadratic_regularisers(g)
        _fuse_relu_maxpool(g)
        _fuse_data_conv_block(g)
        _analyse(g)
        return g

    # -- per-op rules ------------------------------------------------------------------------
    def lower_op(self, op):
        name, a, kw = op.name, op.args, op.kwargs
        A = self.act
        if name in ("aten.detach.default", "aten.detach_.default", "aten.lift_fresh.default"):
            return  # output is a constant
        opname = name.split(".")[1]
        if name in ("aten.add_.Tensor", "aten.sub_.Tensor"):
            return self._inplace_add(op)
        if opname.endswith("_") and not opname.startswith("_"):
            raise UnsupportedGraph(f"in-place op {name} on a parameter-dependent tensor")
        if name in _VIEW_OPS:
            x = A(a[0])
            if name == "aten.expand.default" and tuple(op.out.shape) != tuple(a[0].shape):
                raise UnsupportedGraph("broadcasting expand of a parameter-dependent tensor")
            func, rest = op.func, tuple(a[1:])
            self.alias(x, op.out, lambda t, func=func, rest=rest, kw=dict(kw): func(t, *rest, **kw),
                       full_cover=_VIEW_OPS[name])
            return
        if name == "aten._to_copy.default":
            x = A(a[0])
            okw = {k: v for k, v in kw.items() if k not in ("dtype", "layout", "device", "pin_memory", "non_blocking")
                   and v is not None}
            if okw or not op.out.is_floating_point():
                raise UnsupportedGraph(f"_to_copy with {kw}")
            if op.out.stride() == a[0].stride():
                self.alias(x, op.out, lambda t: t, ident=True)  # a dtype cast is the identity on fp32 tangents/adjoints
            else:
                self.emit("copy", [x], op.out, name)  # cast that also re-lays-out (e.g. of a select view)
            return
        if name == "aten.clone.default":
            x = A(a[0])
            self.emit("copy", [x], op.out, name)  # strided gather into the (usually contiguous) clone
            return
        if name in _UNARY:
            self.emit("unary", [A(a[0])], op.out, name, kind=_UNARY[name],
                      approximate=kw.get("approximate", "none"))
            return
        if name == "aten.pow.Tensor_Scalar":
            self.emit("unary", [A(a[0])], op.out, name, kind="pow", scalar=float(a[1]))
            return
        if name in ("aten.mul.Tensor", "aten.mul.Scalar", "aten.div.Tensor", "aten.div.Scalar"):
            return self._mul_div(op)
        if name in ("aten.add.Tensor", "aten.sub.Tensor", "aten.add.Scalar", "aten.sub.Scalar", "aten.rsub.Scalar"):
            return self._add_sub(op)
        if name in ("aten.sum.default", "aten.mean.default"):
            x = A(a[0])
            scale = 1.0 if name.startswith("aten.sum") else 1.0 / max(1, a[0].numel())
            self.emit("sumall", [x], op.out, name, scale=scale)
            return
        if name in ("aten.sum.dim_IntList", "aten.mean.dim"):
            x = A(a[0])
            dims = a[1] if len(a) > 1 else None
            nd = a[0].dim()
            if dims is None or sorted(d % nd for d in dims) == list(range(nd)):
                scale = 1.0 if name.startswith("aten.sum") else 1.0 / max(1, a[0].numel())
                self.emit("sumall", [x], op.out, name, scale=scale)
                return
            if name == "aten.mean.dim" and nd == 4 and sorted(d % nd for d in dims) == [2, 3] \
                    and a[0].is_contiguous() and kw.get("dtype") is None:
                return self._global_avgpool(op)
            raise UnsupportedGraph(f"partial reduction {name} over dims {dims}")
        if name in ("aten.mm.default", "aten.addmm.default", "aten.bmm.default", "aten.mv.default"):
            return self._gemm(op)
        if name == "aten.convolution.default":
            return self._conv(op)
        if name == "aten.max_pool2d_with_indices.default":
            x = A(a[0])
            self.need_contig(x, "max_pool2d")
            out, idx = op.out
            if not out.is_contiguous():
                raise UnsupportedGraph("max_pool2d: non-contiguous output")
            pair = lambda v, d: tuple(int(q) for q in (v if isinstance(v, (list, tuple)) and len(v) else d)) * (
                2 if isinstance(v, (list, tuple)) and len(v) == 1 else 1)
            kernel = pair(a[1], (1, 1))
            stride = pair(a[2] if len(a) > 2 else [], kernel)
            padding = pair(a[3] if len(a) > 3 else [], (0, 0))
            dilation = pair(a[4] if len(a) > 4 else [], (1, 1))
            # disjoint windows (kernel == stride, no padding / dilation): every input position belongs to at most
            # one window, so the adjoint is a gather that writes each position exactly once (no zero-fill, no atomics)
            disjoint = stride == kernel and padding == (0, 0) and dilation == (1, 1)
            self.emit("maxpool2d", [x], out, name, indices=idx, kernel=kernel, disjoint=disjoint, relu=False)
            return
        if name in _BN_OPS:
            return self._batchnorm(op)
        if name == "aten.native_layer_norm.default":
            return self._layernorm(op)
        if name in ("aten._softmax.default", "aten._log_softmax.default"):
            x = A(a[0])
            dim = a[1] % a[0].dim()
            if dim != a[0].dim() - 1:
                raise UnsupportedGraph("softmax over a non-last dim")
            self.need_contig(x, name)
            self.emit("softmax" if name == "aten._softmax.default" else "logsoftmax", [x], op.out, name)
            return
        if name == "aten.nll_loss_forward.default":
            x = A(a[0])
            target, weight, reduction, ignore_index = a[1], a[2], a[3], a[4]
            if weight is not None:
                raise UnsupportedGraph("nll_loss with class weights")
            if a[0].dim() != 2:
                raise UnsupportedGraph("nll_loss on non-2D input")
            self.need_contig(x, name)
            check = lambda target=target, ii=ignore_index: bool((target == ii).any())
            if check():
                raise UnsupportedGraph("nll_loss with ignored targets")
            self.validators.append((check, "nll_loss with ignored targets"))   # re-run when a cached plan is reused
            out = op.out[0]
            scale = {0: 1.0, 1: 1.0 / a[0].shape[0], 2: 1.0}[reduction]
            self.emit("nll", [x], out, name, target=target, reduction=reduction, scale=scale)
            return
        if name == "aten.binary_cross_entropy_with_logits.default":
            x = A(a[0])
            if A(a[1]) is not None:
                raise UnsupportedGraph("BCE with parameter-dependent targets")
            weight = a[2] if len(a) > 2 else None
            pos_weight = a[3] if len(a) > 3 else None
            reduction = a[4] if len(a) > 4 else 1
            if weight is not None or pos_weight is not None or reduction != 1:
                raise UnsupportedGraph("BCE-with-logits variant")
            self.need_contig(x, name)
            self.emit("bce_logits", [x], op.out, name, target=a[1])
            return
        if name == "aten.embedding.default":
            w = A(a[0])
            if w is None or w.parent is not None or w.param_index is None:
                raise UnsupportedGraph("embedding of a non-parameter table")
            padding_idx = a[2] if len(a) > 2 else -1
            self.emit("embedding", [w], op.out, name, indices=a[1], padding_idx=padding_idx)
            return
        if name == "aten.constant_pad_nd.default":
            x = A(a[0])
            pads = list(a[1])
            if len(a) > 2 and float(a[2]) != 0.0:
                pass   # constant fill value does not matter: it has zero tangent
            nd = a[0].dim()
            out = self._new(op.out)                      # root: buffers stay zero outside the interior
            interior = lambda t, pads=pads, nd=nd, shape=tuple(a[0].shape): _narrow_interior(t, pads, nd, shape)
            inner = self.alias(out, interior(op.out), interior, full_cover=False)
            n = Node("copy", [x], inner, {}, src=name)
            self.nodes.append(n)
            return
        if name == "aten.avg_pool2d.default":
            x = A(a[0])
            kernel = list(a[1])
            stride = list(a[2]) if len(a) > 2 and a[2] else kernel
            padding = list(a[3]) if len(a) > 3 else [0, 0]
            ceil_mode = bool(a[4]) if len(a) > 4 else False
            count_include_pad = bool(a[5]) if len(a) > 5 else True
            divisor = a[6] if len(a) > 6 else None
            if len(kernel) == 1:
                kernel = kernel * 2
            if len(stride) == 1:
                stride = stride * 2
            if len(padding) == 1:
                padding = padding * 2
            if ceil_mode:
                raise UnsupportedGraph("avg_pool2d with ceil_mode")
            self.need_contig(x, name)
            if a[0].dim() != 4 or not op.out.is_contiguous():
                raise UnsupportedGraph("avg_pool2d: only contiguous NCHW")
            # count_include_pad=False: a window is divided by its taps inside the image (only windows that reach into
            # the padding differ from the constant divisor); a divisor override takes precedence, as in aten
            exclude_pad = not count_include_pad and any(padding) and not divisor
            # (no constant divisor on such a node: a rule that ignored exclude_pad would fail instead of using k*k)
            self.emit("avgpool2d", [x], op.out, name, kernel=tuple(kernel), stride=tuple(stride), padding=tuple(padding),
                      divisor=None if exclude_pad else (float(divisor) if divisor else float(kernel[0] * kernel[1])),
                      exclude_pad=exclude_pad)
            return
        if name == "aten.cat.default":
            return self._cat(op)
        if name == "aten.native_dropout.default":
            x = A(a[0])
            out, mask = op.out
            p = float(a[1])
            fn = lambda mask=mask, dt=(a[0].dtype if a[0].dtype == torch.float64 else torch.float32), p=p: mask.to(dt) * (1.0 / (1.0 - p))
            self.emit("mulc", [x], out, name, const=fn(), const_fn=fn, const_srcs=[mask], scalar=None)
            return
        raise UnsupportedGraph(f"no second-order rule for {name}")

    def _mul_div(self, op):
        name, a = op.name, op.args
        x, y = self.act(a[0]), self.act(a[1])
        is_div = ".div" in name
        if x is not None and y is not None:
            if is_div:
                raise UnsupportedGraph("division of two parameter-dependent tensors")
            if tuple(a[0].shape) != tuple(a[1].shape) or a[0].stride() != a[1].stride():
                raise UnsupportedGraph("product of parameter-dependent tensors with different shapes/layout")
            self.emit("mul2", [x, y], op.out, name)
            return
        if x is None:
            if is_div:
                raise UnsupportedGraph("constant / parameter-dependent tensor")
            x, c = y, a[0]
        else:
            c = a[1]
        if isinstance(c, torch.Tensor) and c.requires_grad and not is_div and tuple(c.shape) == tuple(x.base.shape) \
                and c.stride() == x.base.stride() and tuple(op.out.shape) == tuple(c.shape):
            u = self.boundary(c)
            self.emit("mul2", [x, u] if c is a[1] else [u, x], op.out, name)
            return
        if isinstance(c, torch.Tensor):
            if tuple(x.base.shape) != tuple(op.out.shape):
                raise UnsupportedGraph("broadcast of the parameter-dependent factor")

            def fn(c=c, is_div=is_div, shape=tuple(op.out.shape)):
                cc = c.detach()
                cc = cc if cc.dtype == torch.float64 else cc.to(torch.float32)  # fp64 only in the CPU rule tests
                if is_div:
                    cc = 1.0 / cc
                if tuple(cc.shape) != shape:
                    cc = cc.expand(shape)
                return cc.contiguous()

            # const_fn / const_srcs: how to rebuild the constant when a cached plan serves new values (plan.rebind)
            self.emit("mulc", [x], op.out, name, const=fn(), const_fn=fn, const_srcs=[c], scalar=None)
        else:
            s = float(c)
            self.emit("unary", [x], op.out, name, kind="scale", scalar=(1.0 / s if is_div else s))

    def _add_sub(self, op):
        name, a, kw = op.name, op.args, op.kwargs
        alpha = float(kw.get("alpha", 1))
        sub = ".sub" in name
        rsub = "rsub" in name
        x, y = self.act(a[0]), self.act(a[1])
        sx, sy = 1.0, (-alpha if sub else alpha)
        if rsub:
            sx, sy = -1.0, alpha
        if x is not None and y is not None:
            if tuple(a[0].shape) != tuple(a[1].shape):
                raise UnsupportedGraph(f"broadcasting add of parameter-dependent tensors {a[0].shape} + {a[1].shape}")
            self.emit("add2", [x, y], op.out, name, sa=sx, sb=sy)
            return
        v, s = (x, sx) if x is not None else (y, sy)
        if tuple(v.base.shape) != tuple(op.out.shape):
            raise UnsupportedGraph("broadcast of the parameter-dependent addend")
        c = a[1] if x is not None else a[0]
        if isinstance(c, torch.Tensor) and c.requires_grad and tuple(c.shape) == tuple(op.out.shape) \
                and c.stride() == v.base.stride():
            u = self.boundary(c)
            self.emit("add2", [x, u] if x is not None else [u, y], op.out, name, sa=sx, sb=sy)
            return
        if s == 1.0 and op.out.stride() == v.base.stride():
            # y = x + const: identity on tangents and adjoints.  The output is a fresh tensor in the
            # forward but aliases x's second-order buffers.
            self.alias(v, op.out, lambda t: t, ident=True)
        else:
            self.emit("unary", [v], op.out, name, kind="scale", scalar=s)

    _READS_INPUT_BASE = {"unary": (0,), "mul2": (0, 1), "softmax": (0,), "logsoftmax": (0,), "bce_logits": (0,)}

    def _inplace_add(self, op):
        """``x += y`` (residual connections written in place, reference
        examples/learning_to_reweight/model.py:49).  Lowered as a functional add whose result takes over the
        tensor object; refused if an already-recorded rule still needs the overwritten values."""
        name, a, kw = op.name, op.args, op.kwargs
        alpha = float(kw.get("alpha", 1))
        sb = -alpha if ".sub_" in name else alpha
        x, y = self.act(a[0]), self.act(a[1])
        if x is not None and x.parent is not None:
            raise UnsupportedGraph("in-place add into a view of a parameter-dependent tensor")
        if x is not None:
            for n in self.nodes:
                for k in self._READS_INPUT_BASE.get(n.op, ()):
                    if n.ins[k] is not None and n.ins[k].root is x:
                        raise UnsupportedGraph("in-place add overwrites an activation an earlier op still needs")
        if y is not None and tuple(a[0].shape) != tuple(a[1].shape):
            raise UnsupportedGraph("broadcasting in-place add")
        if x is not None and y is not None:
            self.emit("add2", [x, y], op.out, name, sa=1.0, sb=sb)       # re-binds id(tensor) to the new value
        elif x is not None:
            pass                                                            # x += const: same tangents
        else:
            if sb == 1.0 and a[0].stride() == a[1].stride():
                self.alias(y, op.out, lambda t: t, ident=True)
            else:
                self.emit("unary", [y], op.out, name, kind="scale", scalar=sb)

    def _gemm(self, op):
        name, a, kw = op.name, op.args, op.kwargs
        if name == "aten.addmm.default":
            bias_t, A_t, B_t = a
            beta, alpha = float(kw.get("beta", 1)), float(kw.get("alpha", 1))
            if beta != 1 or alpha != 1:
                raise UnsupportedGraph("addmm with alpha/beta != 1")
        else:
            bias_t, (A_t, B_t) = None, a[:2]
        bias = self.act(bias_t) if bias_t is not None else None
        if bias is not None and (bias.base.dim() != 1 or bias.base.shape[0] != op.out.shape[-1]):
            raise UnsupportedGraph("addmm bias that is not a length-N vector")
        va = self.act(A_t) or self.boundary(A_t)
        vb = self.act(B_t) or self.boundary(B_t)
        self.emit("gemm", [va, vb, bias], op.out, name, A=A_t, B=B_t, mv=(name == "aten.mv.default"))

    def _conv(self, op):
        a = op.args
        x_t, w_t, b_t, stride, padding, dilation, transposed, output_padding, groups = a
        if transposed:
            raise UnsupportedGraph("transposed convolution")
        if x_t.dim() != 4:
            raise UnsupportedGraph("only 2-D convolutions")
        x, w, b = self.act(x_t), self.act(w_t), self.act(b_t) if b_t is not None else None
        if x is not None and not x.base.is_contiguous():
            # a strided view (e.g. x[:, :, 1:, 1:]) is gathered into a contiguous value first; the kernels take NCHW
            src, x_t = x_t, x_t.detach().contiguous()
            self.derived.append((x_t, src))          # refreshed from the new call's view when a cached plan is reused
            x = self.emit("copy", [x], x_t, op.name + " (contiguous input)").out
        for v, what in ((x, "conv input"), (w, "conv weight")):
            if v is not None:
                self.need_contig(v, what)
        if not op.out.is_contiguous():
            raise UnsupportedGraph("conv output is not NCHW-contiguous (channels_last?)")
        self.emit("conv2d", [x, w, b], op.out, op.name, X=x_t, W=w_t, stride=tuple(stride), padding=tuple(padding),
                  dilation=tuple(dilation), groups=int(groups))

    def _cat(self, op):
        """``torch.cat``: the output is a root value and every parameter-dependent input is copied into its slice of
        it (a ``narrow`` alias).  Slices of constant inputs are never written, so their tangents stay zero."""
        a = op.args
        ts = list(a[0])
        dim = (a[1] if len(a) > 1 else 0) % op.out.dim()
        if not op.out.is_contiguous():
            raise UnsupportedGraph("cat: non-contiguous output")
        out = self._new(op.out)
        off = 0
        for t in ts:
            if t.dim() == 1 and t.numel() == 0:
                continue                                  # legacy empty operand: takes no slice
            x = self.act(t)
            n = t.shape[dim]
            if x is not None:
                region = lambda u, dim=dim, off=off, n=n: u.narrow(dim, off, n)
                self.nodes.append(Node("copy", [x], self.alias(out, region(op.out), region, full_cover=False), {},
                                       src=op.name))
            off += n

    def _global_avgpool(self, op):
        """``x.mean((-2, -1))`` of a contiguous NCHW tensor (global average pooling) as an ``avgpool2d`` node whose
        window is the whole plane; without keepdim the output is a view of the pooled [N, C, 1, 1] value."""
        x_t, out = op.args[0], op.out
        x = self.act(x_t)
        Nn, Cc, H, W = x_t.shape
        keep = out.dim() == 4
        pooled = out if keep else out.view(Nn, Cc, 1, 1)
        attrs = dict(kernel=(H, W), stride=(H, W), padding=(0, 0), divisor=float(H * W), exclude_pad=False)
        n = self.emit("avgpool2d", [x], pooled, op.name, **attrs)
        if not keep:
            self.alias(n.out, out, lambda t, shape=tuple(out.shape): t.view(shape))

    def _batchnorm(self, op):
        name, a = op.name, op.args
        x_t, g_t, b_t = a[0], a[1], a[2]
        if name in ("aten.native_batch_norm.default", "aten._native_batch_norm_legit.default"):
            training, eps = a[5], a[7]
        elif name in ("aten._native_batch_norm_legit_no_stats.default", "aten._native_batch_norm_legit.no_stats"):
            training, eps = a[3], a[5]
        elif name in ("aten.cudnn_batch_norm.default", "aten.miopen_batch_norm.default"):
            training, eps = a[5], a[7]
        elif name == "aten._batch_norm_with_update.default":
            training, eps = True, a[6]
        else:  # pragma: no cover
            raise UnsupportedGraph(name)
        if not training:
            raise UnsupportedGraph("batch_norm in eval mode (running statistics)")
        x = self.act(x_t)
        if x is None:
            raise UnsupportedGraph("batch_norm of a constant input with parameter-dependent affine")
        self.need_contig(x, "batch_norm")
        out = op.out[0]
        if x_t.dim() != 4 or not out.is_contiguous():
            raise UnsupportedGraph("batch_norm: only contiguous NCHW")
        self.emit("batchnorm", [x, self.act(g_t) if g_t is not None else None,
                                self.act(b_t) if b_t is not None else None], out, name, X=x_t, gamma=g_t,
                  eps=float(eps))

    def _layernorm(self, op):
        a = op.args
        x_t, nshape, g_t, b_t, eps = a
        x = self.act(x_t)
        if x is None:
            raise UnsupportedGraph("layer_norm of a constant input")
        if len(nshape) != 1:
            raise UnsupportedGraph("layer_norm over more than the last dim")
        self.need_contig(x, "layer_norm")
        out = op.out[0]
        self.emit("layernorm", [x, self.act(g_t) if g_t is not None else None,
                                self.act(b_t) if b_t is not None else None], out, op.name, X=x_t, gamma=g_t,
                  eps=float(eps))


def _fold_quadratic_regularisers(g: Graph):
    """Fold ``c * sum((w_i - const)^2)`` loss terms (weight decay, iMAML proximal term, reference
    examples/implicit_maml/main.py:87-92) into one ``diagshift`` node per coefficient:
    ``at_w += 2c * t_w``.  The un-folded form costs three element-wise passes over every parameter and
    ~6 launches per parameter tensor per iteration (RoBERTa: 201 tensors); the curvature of such a term is
    exactly ``2c I`` (SURVEY.md Appendix B, last row), so nothing but that AXPY is needed.

    A term is folded only if the path from its ``sum`` to the loss is affine (add / scale by constants)
    and every value on it has a single consumer; otherwise it is left to the generic rules."""
    root_of = lambda v: v.root
    consumers: Dict[int, List[Tuple[Node, int]]] = {}
    for n in g.nodes:
        for k, v in enumerate(n.ins):
            if v is not None:
                consumers.setdefault(id(root_of(v)), []).append((n, k))
    producer = {id(n.out): n for n in g.nodes if n.out is not None}
    loss_root = g.loss.root

    def ident_chain_to_param(v: Val) -> Optional[Val]:
        while v.parent is not None:
            if not v.ident:
                return None
            v = v.parent
        return v if v.param_index is not None else None

    def param_of(x: Val):
        """(param, theta, s_theta) if x == param (+ s_theta * theta with theta an upper-dependent boundary)."""
        p = ident_chain_to_param(x)
        if p is not None:
            return p, None, 0.0
        n = producer.get(id(x))
        if n is None or n.op != "add2" or len(consumers.get(id(x.root), [])) != 1:
            return None
        for pv, uv, sp, su in ((n.ins[0], n.ins[1], n.attrs["sa"], n.attrs["sb"]),
                               (n.ins[1], n.ins[0], n.attrs["sb"], n.attrs["sa"])):
            pp = ident_chain_to_param(pv)
            if pp is not None and sp == 1.0 and uv.boundary and uv.parent is None:
                return pp, uv, float(su)
        return None

    # d loss / d value along an affine single-consumer path (None if the path is not of that form).  Memoised:
    # weight decay written as ``sum(p.pow(2).sum() for p in params)`` is a chain of ~200 adds, and walking it from
    # every term is quadratic (35 ms of a RoBERTa call's prologue).
    to_loss: Dict[int, Optional[float]] = {id(loss_root): 1.0}

    def factor_to_loss(v: Val) -> Optional[float]:
        path: List[Tuple[int, float]] = []
        cur, res = v, None
        while True:
            rid = id(cur.root)
            if rid in to_loss:
                res = to_loss[rid]
                break
            cons = consumers.get(rid, [])
            if len({id(n) for n, _ in cons}) != 1:
                break
            n = cons[0][0]
            if n.op == "unary" and n.attrs.get("kind") in ("scale", "neg"):
                step = -1.0 if n.attrs["kind"] == "neg" else float(n.attrs["scalar"])
            elif n.op == "add2":
                step = float(sum((n.attrs["sa"] if k == 0 else n.attrs["sb"]) for _, k in cons))
            else:
                break
            path.append((rid, step))
            cur = n.out
        else:
            res = None
        if res is None and id(cur.root) not in to_loss:
            to_loss[id(cur.root)] = None
        for rid, step in reversed(path):
            res = None if res is None else res * step
            to_loss[rid] = res
        return res

    folds: List[Tuple[Val, float, Val, Optional[Val], float]] = []   # (param, coef, x, theta, s_theta)
    removed = set()
    quad_only = set()
    for s_node in g.nodes:
        if s_node.op != "sumall":
            continue
        pw = producer.get(id(s_node.ins[0]))
        if pw is None or pw.op != "unary" or pw.attrs.get("kind") != "pow" or pw.attrs.get("scalar") != 2.0:
            continue
        if len(consumers.get(id(pw.out), [])) != 1:
            continue
        x = pw.ins[0]
        got = param_of(x)
        if got is None or tuple(x.base.shape) != tuple(got[0].base.shape):
            continue
        param, theta, s_theta = got
        f = factor_to_loss(s_node.out)
        if f is None:
            continue
        c = float(s_node.attrs["scale"]) * f
        folds.append((param, 2.0 * c, x, theta, s_theta))
        removed.update((id(pw), id(s_node)))
        quad_only.add(id(s_node.out))
    if not folds:
        return
    new_nodes: List[Node] = []
    for n in g.nodes:
        if id(n) in removed:
            continue
        if n.op == "unary" and n.attrs.get("kind") in ("scale", "neg") and id(n.ins[0].root) in quad_only:
            quad_only.add(id(n.out))
            continue
        if n.op == "add2":
            qa, qb = id(n.ins[0].root) in quad_only, id(n.ins[1].root) in quad_only
            if qa and qb:
                quad_only.add(id(n.out))
                continue
            if qa or qb:
                live, s = (n.ins[1], n.attrs["sb"]) if qa else (n.ins[0], n.attrs["sa"])
                n = Node("unary", [live], n.out, {"kind": "scale", "scalar": float(s)}, src=n.src + " (folded)")
        new_nodes.append(n)
    if id(loss_root) in quad_only:
        return   # the loss is nothing but the regulariser: keep the generic form
    # at_target += coef * t_source.  Curvature: target = source = the parameter.  Mixed term of a proximal
    # regulariser c*sum((w + s*theta)^2): d(g.x)/d theta = 2c*s*x, target = theta's adjoint tangent.
    by_coef: Dict[float, List[Tuple[Val, Val, Val]]] = {}
    for param, coef, x, theta, s_theta in folds:
        by_coef.setdefault(coef, []).append((param, param, x))
        if theta is not None:
            by_coef.setdefault(coef * s_theta, []).append((param, theta, None))
            theta.needed = True
    shifts = []
    for coef, items in by_coef.items():
        for is_theta in (False, True):
            sel = [(s_, t_, x_) for s_, t_, x_ in items if (t_.boundary) == is_theta]
            if sel:
                shifts.append(Node("diagshift", [s_ for s_, _, _ in sel], None,
                                   {"coef": coef, "targets": [t_ for _, t_, _ in sel], "xs": [x_ for _, _, x_ in sel]},
                                   src="folded quadratic regulariser" + (" (mixed term)" if is_theta else "")))
    g.nodes = shifts + new_nodes
    g.stats["folded_terms"] = len(folds)


def _analyse(g: Graph):
    """Dead-code elimination from the loss, then adjoint-writer counting (beta / zero-init)."""
    loss = g.loss
    needed_roots = {id(loss.root)}
    loss.root.needed = True
    live: List[Node] = []
    for n in reversed(g.nodes):
        if n.op == "diagshift":
            live.append(n)          # touches parameter slices only
            continue
        if n.out is None or id(n.out.root) not in needed_roots:
            continue
        live.append(n)
        for v in n.ins:
            if v is not None:
                needed_roots.add(id(v.root))
                v.root.needed = True
    live.reverse()
    g.nodes = live
    for n in live:
        if n.op == "poison":
            raise UnsupportedGraph(f"{n.attrs['error']} [{n.src} feeds the lower loss]")
    if not loss.chain_full_cover():
        # e.g. ``per_sample[0]``: the scalar is one element of a larger root buffer; the executor seeds only that
        # element (plan.py) and the root's other elements must stay zero
        loss.root.zero_init = False
    # count adjoint writers per root (parameters: writers of the H.d slice)
    for v in g.values:
        v.writers = 0
    for n in g.nodes:
        for v in n.ins:
            if v is not None:
                v.root.writers += 1
    for n in g.nodes:
        n.beta = []
        for v in n.ins:
            if v is None:
                n.beta.append(0)
                continue
            r = v.root
            # Overwrite only when this is the buffer's single writer and covers it entirely.  Parameter
            # slices (H.d arena) always accumulate into the arena zeroed at the start of the pass -- several
            # of their kernels are split-K / scatter kernels with atomics -- and so do max-pool / embedding
            # scatters.
            scatter = n.op == "embedding" or (n.op == "maxpool2d" and not n.attrs.get("disjoint"))
            single = r.writers == 1 and v.chain_full_cover() and r.param_index is None and not scatter
            if single:
                n.beta.append(0)
            else:
                n.beta.append(1)
                r.zero_init = True
    for p in g.params:
        p.zero_init = True
    for b in g.boundaries:
        if b.parent is None:
            b.zero_init = True    # read only by the epilogue; may have no node writer (folded proximal terms)
    g.stats = {**g.stats, "nodes": len(g.nodes), "values": sum(1 for v in g.values if v.parent is None and v.needed),
               "aliases": sum(1 for v in g.values if v.parent is not None)}


def _fuse_relu_maxpool(g: Graph):
    """ReLU feeding only a max-pool is folded into the pool node: the arg-max of relu(x) sits where x is largest,
    so relu'(x[argmax]) = [pooled output > 0] and the pool rules become
        TF  t_y = [y > 0] * t_x[argmax]        BB/TB  a_x[argmax] += [y > 0] * a_y
    (relu'' = 0: no curvature term).  Removes a full-size element-wise pass over the pre-pool activation in each
    direction -- the pool output is a quarter of it."""
    import os

    if os.environ.get("BB200_NO_RELU_POOL"):
        return
    consumers: Dict[int, int] = {}
    for n in g.nodes:
        for v in n.ins:
            if v is not None:
                consumers[id(v.root)] = consumers.get(id(v.root), 0) + 1
    producer = {id(n.out): n for n in g.nodes if n.out is not None}
    drop = set()
    for p in g.nodes:
        if p.op != "maxpool2d" or p.ins[0] is None or p.ins[0].parent is not None:
            continue
        x = p.ins[0]
        r = producer.get(id(x))
        if r is None or r.op != "unary" or r.attrs.get("kind") != "relu" or consumers.get(id(x), 0) != 1:
            continue
        src = r.ins[0]
        if x is g.loss or x.boundary or src is None or tuple(src.shape) != tuple(x.shape) or not src.base.is_contiguous():
            continue
        p.ins[0] = src
        p.attrs["relu"] = True
        drop.add(id(r))
    if drop:
        g.nodes = [n for n in g.nodes if id(n) not in drop]
        g.stats = {**g.stats, "relu_pool_fused": len(drop)}


def _fuse_data_conv_block(g: Graph):
    """conv3x3(data) -> BatchNorm2d(batch stats) -> [ReLU] -> MaxPool2d(2) of a DATA input becomes one ``convblock`` node
    (csrc/convblock.cu): with a constant input the conv tangent is linear in the direction, so the BatchNorm
    statistics of every pass are products with per-call Gram matrices and only pooled-size arrays are streamed per
    iteration -- the conv-output-sized tangent / adjoint buffers (y, z) are never allocated.
    (First block of reference examples/implicit_maml/models.py:9-24.)  The member nodes stay in ``attrs['members']``:
    the torch interpreter executes them one by one, and the SURVEY 8(d) byte count still sees three layers."""
    import os

    if os.environ.get("BB200_NO_CONVBLOCK"):
        return
    consumers: Dict[int, List[Node]] = {}
    for n in g.nodes:
        for v in n.ins:
            if v is not None:
                consumers.setdefault(id(v.root), []).append(n)
    out_nodes = []
    dropped = set()
    fused = 0
    for n in g.nodes:
        if id(n) in dropped:
            continue
        blk = _match_data_conv_block(g, n, consumers)
        if blk is None:
            out_nodes.append(n)
            continue
        conv, bn, pool = blk
        x, w, b = conv.ins
        gam, bet = bn.ins[1], bn.ins[2]
        conv.beta, bn.beta, pool.beta = [0, 1, 1], [0, 1, 1], [0]   # what _analyse would give the members
        attrs = dict(members=[conv, bn, pool], X=conv.attrs["X"], W=conv.attrs["W"], Y=conv.out.base,
                     padding=conv.attrs["padding"], eps=bn.attrs["eps"], gamma=bn.attrs["gamma"],
                     indices=pool.attrs["indices"], relu=bool(pool.attrs.get("relu")))
        tail = "+batch_norm+relu+max_pool2d" if pool.attrs.get("relu") else "+batch_norm+max_pool2d"
        if x is None:
            node = Node("convblock", [w, b, gam, bet], pool.out, attrs, src="conv3x3(data)" + tail)
        else:
            node = Node("convblock2", [x, w, b, gam, bet], pool.out, attrs, src="conv3x3" + tail)
        conv.out.interp_only = bn.out.interp_only = True
        out_nodes.append(node)
        dropped.update((id(bn), id(pool)))
        fused += 1
    if fused:
        g.nodes = out_nodes
        g.stats = {**g.stats, "conv_blocks_fused": fused}
        # a pooled tangent that only feeds the next fused inner block is written directly as that block's bf16 NHWC
        # TMA operand (64 channels): no fp32 buffer, no pack kernel
        cons: Dict[int, List[Node]] = {}
        for n in g.nodes:
            for v in n.ins:
                if v is not None:
                    cons.setdefault(id(v.root), []).append(n)
        for n in g.nodes:
            if n.op in ("convblock", "convblock2") and n.out.parent is None and n.out.base.shape[1] == 64:
                users = cons.get(id(n.out), [])
                if len(users) == 1 and users[0].op == "convblock2" and users[0].ins[0] is n.out and n.out is not g.loss:
                    n.out.tfmt = "nhwc_bf16"


def _match_data_conv_block(g: Graph, conv: Node, consumers) -> Optional[Tuple[Node, Node, Node]]:
    import os

    if conv.op != "conv2d" or conv.ins[1] is None:
        return None
    at = conv.attrs
    W, X = at["W"], at["X"]
    if (at["groups"] != 1 or tuple(at["stride"]) != (1, 1) or tuple(at["dilation"]) != (1, 1)
            or tuple(W.shape[2:]) != (3, 3) or W.shape[0] > 64):
        return None
    if conv.ins[0] is None:
        if W.shape[1] not in (1, 3):                     # data-input block (convblock.cu)
            return None
    else:
        # inner block (convblock2.cu): bf16-autocast graphs only -- its products run on the TMA tensor-core kernels,
        # whose shape limits (conv_tma.cu bb_conv_tma_ok) apply
        x = conv.ins[0]
        reduced = X.dtype in (torch.bfloat16, torch.float16) and W.dtype in (torch.bfloat16, torch.float16)
        C, O, Wd, WO = W.shape[1], W.shape[0], X.shape[3], conv.out.base.shape[3]
        # 64 -> 64 channels, and a band of 128 + 2(W+2) + 2 pixel rows must fit one TMA box (conv_halo.cu)
        if (os.environ.get("BB200_NO_CONVBLOCK2") or not reduced or x.parent is not None or x.boundary
                or C != 64 or O != 64 or not (4 <= WO <= 61) or Wd != WO
                or tuple(at["padding"]) != (1, 1) or not X.is_contiguous()):
            return None
    def is_param(v):
        # the parameter itself, or its autocast copy (an identity alias: same tangent / adjoint-tangent slices)
        while v is not None and v.parent is not None and v.ident:
            v = v.parent
        return v is not None and v.parent is None and v.param_index is not None

    if not is_param(conv.ins[1]) or (conv.ins[2] is not None and not is_param(conv.ins[2])):
        return None
    y = conv.out
    cons = consumers.get(id(y), [])
    if len(cons) != 1 or cons[0].op != "batchnorm" or cons[0].ins[0] is not y or y is g.loss:
        return None
    bn = cons[0]
    for v in bn.ins[1:]:
        if v is not None and not is_param(v):
            return None
    if bn.attrs["gamma"] is not None and bn.attrs["gamma"].dtype != torch.float32:
        return None
    z = bn.out
    cons = consumers.get(id(z), [])
    if len(cons) != 1 or cons[0].op != "maxpool2d" or cons[0].ins[0] is not z or z is g.loss:
        return None
    pool = cons[0]
    if tuple(pool.attrs.get("kernel", ())) != (2, 2) or not pool.attrs.get("disjoint"):
        return None
    if not (y.base.is_contiguous() and z.base.is_contiguous() and pool.out.base.is_contiguous()):
        return None
    return conv, bn, pool


def lower_tape(tape, fold_quadratic: bool = True) -> Graph:
    return _Lowering(tape).run(fold_quadratic)
