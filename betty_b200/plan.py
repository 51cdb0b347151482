"""Native second-order plan: lowers a recorded tape (ir.py), lays every tangent / adjoint buffer out in
a handful of device arenas, serialises the node list into ``bb_node`` descriptors (csrc/plan.h) and
drives the C executor (csrc/plan.cu).  After construction the K-loop makes no Python-level launches:
``neumann_loop`` / ``cg_loop`` are one C call each (CUDA-graph replay of one iteration).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _native as N
from .arena import ArenaLayout
from .ir import Graph, Node, UnsupportedGraph, Val, _is_dense, lower_tape

BB_MAX_DIMS = 6
OPS = {"unary": 1, "copy": 2, "add2": 3, "mulc": 4, "mul2": 5, "sumall": 6, "gemm": 7, "conv2d": 8,
       "maxpool2d": 9, "batchnorm": 10, "layernorm": 11, "softmax": 12, "logsoftmax": 13, "nll": 14,
       "bce_logits": 15, "embedding": 16, "diagshift": 17, "avgpool2d": 18, "convblock": 19, "convblock2": 20}
UNARY = {"relu": 1, "gelu": 2, "tanh": 3, "sigmoid": 4, "pow": 5, "scale": 6, "neg": 6}
PASS_BB, PASS_TF, PASS_TB = 0, 1, 2

NODE_DTYPE = np.dtype([
    ("op", np.int32), ("kind", np.int32), ("active", np.int32), ("linear", np.int32),
    ("beta", np.int32, (4,)), ("dt", np.int32, (4,)), ("ndim", np.int32), ("pad0", np.int32),
    ("n", np.int64), ("dims", np.int64, (16,)), ("f", np.float64, (4,)),
    ("base", np.uint64, (4,)), ("t", np.uint64, (4,)), ("a", np.uint64, (4,)), ("at", np.uint64, (4,)),
    ("aux", np.uint64, (4,)), ("sizes", np.int64, (BB_MAX_DIMS,)), ("stride", np.int64, (4, BB_MAX_DIMS)),
], align=True)


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return 0
    if t.dtype == torch.bfloat16:
        return 1
    if t.dtype == torch.float16:
        return 2
    raise UnsupportedGraph(f"activation dtype {t.dtype} (only fp32 and bf16 / fp16 autocast are supported)")


def _align(n: int, a: int = 64) -> int:
    return (n + a - 1) // a * a


class HvpPlan:
    def __init__(self, tape, params: Sequence[torch.Tensor], layout: ArenaLayout, d_arena: torch.Tensor,
                 hv_arena: torch.Tensor, cuda_graph: Optional[bool] = None, dry_run: bool = False):
        """``dry_run`` (CPU unit tests only) builds buffers and descriptors but launches nothing."""
        from .engine import settings

        if not dry_run:
            N.require_cuda()
        assert N.lib().bb_node_bytes() == NODE_DTYPE.itemsize, (N.lib().bb_node_bytes(), NODE_DTYPE.itemsize)
        self.dev = d_arena.device
        self.layout, self.d_arena, self.hv_arena = layout, d_arena, hv_arena
        self.use_graph = settings.cuda_graph if cuda_graph is None else cuda_graph
        self.tape = tape                      # keeps the base activations alive
        self.dry_run = dry_run
        self.g: Graph = lower_tape(tape)
        self._keep: List[torch.Tensor] = []   # constants / scratch referenced by raw pointer
        self._derived: list = []              # (constant, thunk recomputing it from the tape's tensors) -- see rebind()
        self._views: dict = {}                # (id(alias value), kind) -> torch view of its root buffer
        self._alloc_buffers()
        self._build_nodes()
        self.launches_per_iter = 0
        self.serves = 1                       # hypergradient calls this plan has served (plan cache, engine.py)
        self.boundary_bases = None            # vid -> upper-dependent tensor of the CURRENT call's forward (after rebind)
        self._locator = None
        if dry_run:
            return
        self.side = torch.cuda.Stream(device=self.dev)
        self.run_pass(PASS_BB)                # delta, once per call (reference: part of in_grad's backward)

    # ------------------------------------------------------------------------------------------
    def _alloc_buffers(self):
        g = self.g
        roots = [v for v in g.values if v.parent is None and (v.needed or v.boundary) and v.param_index is None]
        for v in roots:
            if not _is_dense(v.base):
                raise UnsupportedGraph(f"activation {v} is not dense (strides {v.base.stride()})")
        sizes = {"t": 0, "z": 0, "nz": 0}
        place = {}
        for v in roots:
            n = _align(v.base.numel())
            place[v.vid] = (sizes["t"], sizes["z" if v.zero_init else "nz"])
            if v.tfmt is None:
                sizes["t"] += n
                sizes["z" if v.zero_init else "nz"] += n
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.T = torch.zeros(max(sizes["t"], 1), **f32)
        self.A = {"z": torch.zeros(max(sizes["z"], 1), **f32), "nz": torch.zeros(max(sizes["nz"], 1), **f32)}
        self.AT = {"z": torch.zeros(max(sizes["z"], 1), **f32), "nz": torch.zeros(max(sizes["nz"], 1), **f32)}
        self.zero_bytes = 4 * sizes["z"]
        for v in roots:
            ot, oa = place[v.vid]
            k = "z" if v.zero_init else "nz"
            shape, stride = tuple(v.base.shape), tuple(v.base.stride())
            if v.tfmt == "nhwc_bf16":
                # tangent written by a fused block directly as the next fused block's TMA operand: bf16 padded NHWC
                # [N][H+2][W+2][64], zero border (never written)
                Nn, Cc, Hh, Ww = shape
                assert Cc == 64, shape
                mk = lambda: torch.zeros((Nn, Hh + 2, Ww + 2, 64), dtype=torch.bfloat16, device=self.dev)
                v.t, v.a, v.at = mk(), mk(), mk()       # (single producer each, every interior element overwritten)
                continue
            v.t = torch.as_strided(self.T, shape, stride, ot)
            v.a = torch.as_strided(self.A[k], shape, stride, oa)
            v.at = torch.as_strided(self.AT[k], shape, stride, oa)
        dviews, hviews = self.layout.views(self.d_arena), self.layout.views(self.hv_arena)
        for p in g.params:
            if not p.base.is_contiguous() or p.base.dtype != torch.float32:
                raise UnsupportedGraph("lower parameters must be contiguous fp32 tensors")
            p.t, p.at, p.a = dviews[p.param_index], hviews[p.param_index], None
        # seed dL/dL = 1 through the loss's own alias chain: when the scalar is one element of a larger tensor
        # (``per_sample[0]``) the root's other elements must stay 0; its adjoint tangent stays 0
        g.loss.root.a.zero_()
        self.buf(g.loss, "a").fill_(1.0)
        self.bytes_buffers = 4 * (self.T.numel() + 2 * (self.A["z"].numel() + self.A["nz"].numel()))

    def buf(self, v: Optional[Val], kind: str) -> Optional[torch.Tensor]:
        if v is None:
            return None
        if v.parent is None:
            return getattr(v, kind)
        key = (id(v), kind)             # alias views are asked for several times per consuming node: build them once
        hit = self._views.get(key, self)
        if hit is not self:
            return hit
        b = self.buf(v.parent, kind)
        out = None if b is None else v.viewfn(b)
        self._views[key] = out
        return out

    # ------------------------------------------------------------------------------------------
    def _ptr(self, t: Optional[torch.Tensor]) -> int:
        return 0 if t is None else t.data_ptr()

    def _const(self, t: torch.Tensor, dtype=None, recipe=None) -> torch.Tensor:
        """A constant the descriptors point at.  ``recipe`` (or, for a converted copy of a tape tensor, the conversion
        itself) is remembered so that ``rebind`` can refresh the values in place when the plan is reused."""
        def make(src=t):
            o = src.detach()
            if dtype is not None and o.dtype != dtype:
                o = o.to(dtype)
            return o.to(self.dev).contiguous()

        out = make()
        self._keep.append(out)
        if recipe is not None:
            self._derived.append((out, lambda: make(recipe())))
        elif out.data_ptr() != t.data_ptr():
            self._derived.append((out, make))
        return out

    def _scratch(self, nbytes: int) -> torch.Tensor:
        t = torch.zeros(_align(nbytes, 8) // 8, dtype=torch.float64, device=self.dev)
        self._keep.append(t)
        return t

    def _slot(self, rec, s: int, v: Optional[Val], base_t: Optional[torch.Tensor]):
        """Fill operand slot ``s`` (pointers + dtype); returns the buffer used for stride checks."""
        if base_t is not None:
            rec["base"][s] = base_t.data_ptr()
            rec["dt"][s] = _dt(base_t) if base_t.is_floating_point() else 0
        if v is not None:
            for kind in ("t", "a", "at"):
                b = self.buf(v, kind)
                rec[kind][s] = self._ptr(b)
                if v.root.tfmt is not None:
                    continue            # bf16 padded-NHWC buffers handed from one fused block to the next
                if b is not None and base_t is not None and b.numel() > 1 and tuple(b.stride()) != tuple(base_t.stride()):
                    raise UnsupportedGraph(f"buffer/base stride mismatch for {v}: {b.stride()} vs {base_t.stride()}")

    def _build_nodes(self):
        g = self.g
        recs = np.zeros(len(g.nodes), dtype=NODE_DTYPE)
        for i, n in enumerate(g.nodes):
            r = recs[i]
            r["op"] = OPS[n.op]
            if n.op != "diagshift":   # (its inputs are a parameter list, not operand slots)
                r["active"] = sum(1 << k for k, v in enumerate(n.ins) if v is not None)
                r["pad0"] = sum(1 << k for k, v in enumerate(n.ins) if v is not None and v.root.param_index is None)
                for k, b in enumerate(n.beta[:4]):
                    r["beta"][k] = b
            getattr(self, "_n_" + n.op)(n, r)
        self.recs = recs
        handle = C.c_void_p()
        N.call("bb_plan_create", recs.ctypes.data, len(recs), C.byref(handle))
        self.handle = handle

        def regions(ts):
            ts = [t for t in ts if t is not None and t.numel() > 0]
            ptrs = (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
            nb = (C.c_int64 * len(ts))(*[t.numel() * t.element_size() for t in ts])
            return ptrs, nb, len(ts)

        # scratch of the TMA-fed tensor-core kernels (bf16 operand packs; csrc/gemm_tma.cu, conv_tma.cu): the largest
        # single node's need, since packs never outlive their node
        need = max([self._tma_scratch_bytes(r) for r in recs] + [0])
        if need and not self.dry_run:
            self.tma_scratch = torch.empty(need, dtype=torch.uint8, device=self.dev)
            N.call("bb_plan_set_scratch", self.handle, self.tma_scratch.data_ptr(), need)

        persist = sum(self._tma_persistent_bytes(r) for r in recs)
        if persist and need and not self.dry_run:
            self.tma_persistent = torch.empty(persist, dtype=torch.uint8, device=self.dev)
            N.call("bb_plan_set_persistent", self.handle, self.tma_persistent.data_ptr(), persist)

        # a folded c*I term over EVERY parameter is applied by the K-loop vector kernels (their `shift`) instead of a
        # 12 B/parameter sweep per iteration; the bare H.d product (tests, epilogue) still runs the node
        self.uniform_shift = None
        all_params = {id(p) for p in g.params}
        for i, n in enumerate(g.nodes):
            if n.op == "diagshift" and not any(t.boundary for t in n.attrs["targets"]):
                tg = [id(t) for t in n.attrs["targets"]]
                if len(tg) == len(set(tg)) == len(all_params) and set(tg) == all_params and all(
                        s_ is t_ for s_, t_ in zip(n.ins, n.attrs["targets"])):
                    if not self.dry_run:
                        N.call("bb_plan_set_uniform_shift", self.handle, i, float(n.attrs["coef"]))
                    self.uniform_shift = (i, float(n.attrs["coef"]))
                    break

        zb = [self.A["z"]] if self.zero_bytes else []
        zt = ([self.AT["z"]] if self.zero_bytes else []) + [self.hv_arena]
        for pas, ts in ((PASS_BB, zb), (PASS_TF, []), (PASS_TB, zt)):
            ptrs, nb, cnt = regions(ts)
            N.call("bb_plan_set_zero_regions", self.handle, pas, ptrs, nb, cnt)

    @staticmethod
    def _tma_persistent_bytes(r) -> int:
        """Plan-lifetime pack of a data-input convolution's im2col matrix (csrc/conv_tma.cu run_small_c)."""
        if not (int(r["kind"]) & 1) or int(r["op"]) != OPS["conv2d"]:
            return 0
        Nn, Cc, H, W, O, KH, KW, HO, WO = (int(x) for x in r["dims"][0:9])
        ckk, act = Cc * KH * KW, int(r["active"])
        if not (act & 1) and (act & 2) and 8 <= ckk <= 64 and 32 <= O <= 128 and Nn * HO * WO >= 128:
            return 2 * Nn * HO * WO * _align(ckk, 8) + 512
        unit = all(int(x) == 1 for x in (r["dims"][9], r["dims"][10], r["dims"][13], r["dims"][14]))
        if unit and KH * KW <= 9 and 32 <= Cc <= 64 and 32 <= O <= 64 and 4 <= WO <= 64 and W <= 128:
            return 2 * 64 * Nn * (H * W + HO * WO) + 1024      # NHWC bf16 packs of x and of the base adjoint a_y
        return 0

    @staticmethod
    def _tma_scratch_bytes(r) -> int:
        """Upper bound of the bf16 pack bytes one node's launch needs (mirrors the checks in gemm_tma.cu / conv_tma.cu)."""
        if not (int(r["kind"]) & 1):
            return 0
        if int(r["op"]) == OPS["gemm"]:
            M, Nn, K, batch = (int(x) for x in r["dims"][0:4])
            pad = lambda a, b: batch * (a + 8) * (b + 8)
            # packs live for the whole node (TB: both adjoints, both weights, both inputs) and the launcher's
            # admission check counts either layout of every operand of the launch at hand
            return 2 * 4 * (pad(M, K) + pad(Nn, K) + pad(M, Nn)) + 16384
        if int(r["op"]) == OPS["conv2d"]:
            Nn, Cc, H, W, O, KH, KW, HO, WO = (int(x) for x in r["dims"][0:9])
            unit = all(int(x) == 1 for x in (r["dims"][9], r["dims"][10], r["dims"][13], r["dims"][14]))
            ckk, act = Cc * KH * KW, int(r["active"])
            if not (act & 1) and (act & 2) and 8 <= ckk <= 64 and 32 <= O <= 128 and Nn * HO * WO >= 128:
                kp, opad = _align(ckk, 8), _align(O, 64)      # data-input layer: im2col matrix + packed at_y
                return 2 * Nn * HO * WO * (kp + opad) + 2 * (O + 8) * (kp + 8) + 16384 + 8192
            if not (unit and KH * KW <= 9 and 32 <= Cc <= 64 and 32 <= O <= 64 and 4 <= WO <= 64 and W <= 128):
                return 0          # bb_conv_tma_ok() declines: software-staged / SIMT kernels, no packs
            cp, op = _align(Cc, 64), _align(O, 64)
            acts = 2 * Nn * H * W * cp + 2 * Nn * HO * WO * op
            return 2 * (acts + 4 * op * KH * KW * cp) + 16384
        return 0

    # ---- per-op descriptor builders -----------------------------------------------------------
    def _ew_layout(self, r, out: Val, operands: List[Optional[torch.Tensor]]):
        """operands: buffers (or const tensors) for slots 0,1,2; slot 3 is the output buffer."""
        ob = self.buf(out, "t")
        shape = tuple(ob.shape)
        if len(shape) > BB_MAX_DIMS:
            raise UnsupportedGraph(f"element-wise op on a {len(shape)}-d tensor")
        tens = list(operands) + [ob]
        linear = _is_dense(ob)
        for t in tens:
            if t is None:
                continue
            if tuple(t.shape) != shape:
                raise UnsupportedGraph(f"element-wise operand shape {tuple(t.shape)} != {shape}")
            if ob.numel() > 1 and tuple(t.stride()) != tuple(ob.stride()):
                linear = False
        r["linear"] = int(linear)
        r["ndim"] = max(len(shape), 1)
        r["n"] = ob.numel()
        for d, sz in enumerate(shape):
            r["sizes"][d] = sz
        if not shape:
            r["sizes"][0] = 1
        for s, t in enumerate(tens):
            if t is None:
                continue
            for d, st in enumerate(t.stride()):
                r["stride"][s][d] = st

    def _n_diagshift(self, n: Node, r):
        from .arena import ChunkTable

        ts = [self.buf(p, "t") for p in n.ins]                     # sources: parameter tangents
        ats = [self.buf(t, "at") for t in n.attrs["targets"]]      # targets: H.d slices, or a boundary's at
        for a, b in zip(ts, ats):
            if not (a.is_contiguous() and b.is_contiguous() and a.numel() == b.numel()):
                raise UnsupportedGraph("folded quadratic term over a non-contiguous tensor")
        tab = ChunkTable([t.data_ptr() for t in ts], [t.data_ptr() for t in ats], [t.numel() for t in ts], self.dev,
                         keep=(ts, ats))
        self._keep.append(tab.dev)
        r["aux"][0] = tab.ptr
        r["dims"][0] = tab.n
        r["f"][0] = n.attrs["coef"]
        r["n"] = sum(t.numel() for t in ts)

    def _n_unary(self, n: Node, r):
        x = n.ins[0]
        r["kind"] = UNARY[n.attrs["kind"]]
        if n.attrs["kind"] == "gelu" and n.attrs.get("approximate", "none") != "none":
            raise UnsupportedGraph("tanh-approximated GELU")
        r["f"][0] = -1.0 if n.attrs["kind"] == "neg" else float(n.attrs.get("scalar") or 0.0)
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)
        self._ew_layout(r, n.out, [self.buf(x, "t"), None, None])

    def _n_copy(self, n: Node, r):
        x = n.ins[0]
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)
        self._ew_layout(r, n.out, [self.buf(x, "t"), None, None])

    def _n_add2(self, n: Node, r):
        a, b = n.ins
        r["f"][1], r["f"][2] = n.attrs["sa"], n.attrs["sb"]
        self._slot(r, 0, a, a.base)
        self._slot(r, 1, b, b.base)
        self._slot(r, 3, n.out, None)
        self._ew_layout(r, n.out, [self.buf(a, "t"), self.buf(b, "t"), None])

    def _n_mulc(self, n: Node, r):
        x = n.ins[0]
        c = self._const(n.attrs["const"], torch.float32, recipe=n.attrs.get("const_fn"))
        r["aux"][0] = c.data_ptr()
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)
        self._ew_layout(r, n.out, [self.buf(x, "t"), None, c])

    def _n_mul2(self, n: Node, r):
        a, b = n.ins
        self._slot(r, 0, a, a.base)
        self._slot(r, 1, b, b.base)
        self._slot(r, 3, n.out, None)
        self._ew_layout(r, n.out, [self.buf(a, "t"), self.buf(b, "t"), None])

    def _n_sumall(self, n: Node, r):
        x = n.ins[0]
        xb = self.buf(x, "t")
        if not _is_dense(xb):
            raise UnsupportedGraph("full reduction of a non-dense tensor")
        r["n"] = xb.numel()
        r["f"][0] = n.attrs["scale"]
        r["aux"][0] = self._scratch(8 * (2 * 132 + 2)).data_ptr()   # kRedMaxGrid = 2 x BB_SM_COUNT partials
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)

    def _n_gemm(self, n: Node, r):
        A_t, B_t = n.attrs["A"], n.attrs["B"]
        a, b, bias = n.ins
        out = n.out.base
        if n.attrs["mv"]:
            M, K = A_t.shape
            Nn, batch = 1, 1
            sa = (A_t.stride(0), A_t.stride(1), 0)
            sb = (B_t.stride(0), 0, 0)
            sc = (out.stride(0), 0, 0)
        elif A_t.dim() == 2:
            M, K = A_t.shape
            Nn, batch = B_t.shape[1], 1
            sa = (A_t.stride(0), A_t.stride(1), 0)
            sb = (B_t.stride(0), B_t.stride(1), 0)
            sc = (out.stride(0), out.stride(1), 0)
        else:
            batch, M, K = A_t.shape
            Nn = B_t.shape[2]
            sa = (A_t.stride(1), A_t.stride(2), A_t.stride(0))
            sb = (B_t.stride(1), B_t.stride(2), B_t.stride(0))
            sc = (out.stride(1), out.stride(2), out.stride(0))
        r["dims"][0:4] = (M, Nn, K, batch)
        # bf16-autocast graph: this product was computed from bf16 operands by the reference too, so the
        # tensor-core (bf16 x bf16 -> fp32) kernel keeps the 1e-2 parity bar; fp32 graphs stay on exact fp32
        r["kind"] = int(A_t.dtype in (torch.bfloat16, torch.float16) or B_t.dtype in (torch.bfloat16, torch.float16))
        for d in range(3):
            r["stride"][0][d], r["stride"][1][d], r["stride"][3][d] = sa[d], sb[d], sc[d]
        self._slot(r, 0, a, A_t)
        self._slot(r, 1, b, B_t)
        self._slot(r, 3, n.out, None)
        if bias is not None:
            bb = self.buf(bias, "t")
            r["stride"][2][0] = bb.stride(0)
            self._slot(r, 2, bias, None)

    def _n_conv2d(self, n: Node, r):
        x, w, b = n.ins
        X, W = n.attrs["X"], n.attrs["W"]
        if n.attrs["groups"] != 1:
            raise UnsupportedGraph("grouped / depthwise convolution")
        if not X.is_contiguous() or not W.is_contiguous():
            raise UnsupportedGraph("conv operands must be NCHW-contiguous")
        Nn, Cc, H, Wd = X.shape
        O, _, KH, KW = W.shape
        _, _, HO, WO = n.out.base.shape
        (sh, sw), (ph, pw), (dh, dw) = n.attrs["stride"], n.attrs["padding"], n.attrs["dilation"]
        r["dims"][0:15] = (Nn, Cc, H, Wd, O, KH, KW, HO, WO, sh, sw, ph, pw, dh, dw)
        r["kind"] = int(X.dtype in (torch.bfloat16, torch.float16) or W.dtype in (torch.bfloat16, torch.float16))  # reduced-precision graph -> tensor cores allowed
        self._slot(r, 0, x, X)
        self._slot(r, 1, w, W)
        self._slot(r, 2, b, None)
        self._slot(r, 3, n.out, None)

    def _n_maxpool2d(self, n: Node, r):
        x = n.ins[0]
        idx = n.attrs["indices"]
        Nn, Cc, H, W = x.base.shape
        _, _, HO, WO = n.out.base.shape
        kh, kw = n.attrs.get("kernel", (1, 1))
        r["dims"][0:9] = (Nn * Cc, H * W, HO * WO, H, W, HO, WO, kh, kw)
        # kind bit 0: ReLU folded in (mask = pooled base output > 0); bit 1: disjoint windows -> gather-form adjoint
        r["kind"] = int(bool(n.attrs.get("relu"))) | (int(bool(n.attrs.get("disjoint"))) << 1)
        r["aux"][0] = self._const(idx, torch.int64).data_ptr()
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, n.out.base)

    def _n_convblock(self, n: Node, r):
        """Fused data-input conv3x3 -> BatchNorm -> [ReLU] -> MaxPool2d(2) (csrc/convblock.cu; slot map there)."""
        w, b, gam, bet = n.ins
        X, W, Y = n.attrs["X"], n.attrs["W"], n.attrs["Y"]
        Nn, Cc, H, Wd = X.shape
        O = W.shape[0]
        _, _, HO, WO = Y.shape
        _, _, HP, WP = n.out.base.shape
        ph, pw = n.attrs["padding"]
        r["dims"][0:16] = (Nn, Cc, H, Wd, O, 3, 3, HO, WO, 1, 1, ph, pw, HP, WP, int(n.attrs["relu"]))
        r["f"][0] = n.attrs["eps"]
        # kind: bit 0 reduced precision, bit 2: t of q is bf16 padded NHWC, bit 3: so are a / at of q
        r["kind"] = int(X.dtype in (torch.bfloat16, torch.float16)) | (12 if n.out.tfmt == "nhwc_bf16" else 0)
        if not (X.is_contiguous() and Y.is_contiguous()):
            raise UnsupportedGraph("convblock operands must be NCHW-contiguous")
        self._slot(r, 0, w, None)
        self._slot(r, 1, b, None)
        g_t = n.attrs["gamma"]
        self._slot(r, 2, gam, g_t)                       # base[2] = gamma values (fp32 parameter)
        self._slot(r, 3, n.out, n.out.base)
        r["base"][0], r["dt"][0] = X.data_ptr(), _dt(X)
        r["base"][1], r["dt"][1] = Y.data_ptr(), _dt(Y)
        nbytes = int(N.lib().bb_convblock_ws_bytes(Nn, Cc, H, Wd, O, HO, WO, HP, WP))
        ws = torch.zeros(nbytes // 8 + 1, dtype=torch.float64, device=self.dev)
        self._keep.append(ws)
        r["aux"][0] = ws.data_ptr()
        r["aux"][1] = self._ptr(self.buf(bet, "t"))
        r["aux"][2] = self._ptr(self.buf(bet, "at"))
        r["aux"][3] = self._const(n.attrs["indices"], torch.int64).data_ptr()

    def _n_convblock2(self, n: Node, r):
        """Fused inner conv3x3 -> BatchNorm -> [ReLU] -> MaxPool2d(2) of a bf16 graph (csrc/convblock2.cu; slot map there)."""
        x, w, b, gam, bet = n.ins
        X, W, Y = n.attrs["X"], n.attrs["W"], n.attrs["Y"]
        Nn, Cc, H, Wd = X.shape
        O = W.shape[0]
        _, _, HO, WO = Y.shape
        _, _, HP, WP = n.out.base.shape
        ph, pw = n.attrs["padding"]
        r["dims"][0:16] = (Nn, Cc, H, Wd, O, 3, 3, HO, WO, 1, 1, ph, pw, HP, WP, int(n.attrs["relu"]))
        r["f"][0] = n.attrs["eps"]
        if not (X.is_contiguous() and Y.is_contiguous() and W.is_contiguous()):
            raise UnsupportedGraph("convblock2 operands must be contiguous")
        # kind: bit 0 reduced precision, bit 1: t of x_in is bf16 NHWC, bit 2: t of q is bf16 NHWC
        r["kind"] = 1 | (2 if x.tfmt == "nhwc_bf16" else 0) | (4 if n.out.tfmt == "nhwc_bf16" else 0)
        for s_, v in ((0, x), (1, w), (2, gam), (3, n.out)):
            if v is None:
                continue
            for kind in ("t", "a", "at"):
                r[kind][s_] = self._ptr(self.buf(v, kind))
        r["base"][0], r["dt"][0] = X.data_ptr(), _dt(X)
        r["base"][1], r["dt"][1] = W.data_ptr(), _dt(W)
        g_t = n.attrs["gamma"]
        r["base"][2] = g_t.data_ptr() if g_t is not None else 0
        r["base"][3], r["dt"][3] = n.out.base.data_ptr(), _dt(n.out.base)
        nbytes = int(N.lib().bb_convblock2_ws_bytes(Nn, Cc, H, Wd, O, HO, WO, HP, WP))
        ws = torch.zeros(nbytes // 8 + 1, dtype=torch.float64, device=self.dev)
        self._keep.append(ws)
        r["aux"][0] = ws.data_ptr()
        r["aux"][1] = self._const(n.attrs["indices"], torch.int64).data_ptr()
        r["aux"][2] = Y.data_ptr()
        r["ndim"] = _dt(Y)
        ptrs = [self._ptr(self.buf(b, "t")), self._ptr(self.buf(b, "at")), self._ptr(self.buf(bet, "t")),
                self._ptr(self.buf(bet, "at"))]
        for k, pv in enumerate(ptrs):
            r["stride"][0][k] = np.int64(np.uint64(pv).astype(np.int64)) if pv >= 2 ** 63 else pv

    def _n_avgpool2d(self, n: Node, r):
        x = n.ins[0]
        Nn, Cc, H, W = x.base.shape
        _, _, HO, WO = n.out.base.shape
        (kh, kw), (sh, sw), (ph, pw) = n.attrs["kernel"], n.attrs["stride"], n.attrs["padding"]
        r["dims"][0:11] = (Nn * Cc, H, W, HO, WO, kh, kw, sh, sw, ph, pw)
        r["f"][0] = 1.0 / n.attrs["divisor"]
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)

    def _n_batchnorm(self, n: Node, r):
        x, gv, bv = n.ins
        X = n.attrs["X"]
        Nn, Cc, H, W = X.shape
        r["dims"][0:3] = (Nn, Cc, H * W)
        r["f"][0] = n.attrs["eps"]
        r["aux"][0] = self._scratch(8 * 16 * Cc).data_ptr()
        self._slot(r, 0, x, X)
        gam = n.attrs["gamma"]
        if gam is not None:
            self._slot(r, 1, gv, self._const(gam, torch.float32) if gam.dtype != torch.float32 else gam)
        self._slot(r, 2, bv, None)
        self._slot(r, 3, n.out, None)

    def _n_layernorm(self, n: Node, r):
        x, gv, bv = n.ins
        X = n.attrs["X"]
        D = X.shape[-1]
        r["dims"][0:2] = (X.numel() // D, D)
        r["f"][0] = n.attrs["eps"]
        self._slot(r, 0, x, X)
        gam = n.attrs["gamma"]
        if gam is not None:
            self._slot(r, 1, gv, self._const(gam, torch.float32) if gam.dtype != torch.float32 else gam)
        self._slot(r, 2, bv, None)
        self._slot(r, 3, n.out, None)

    def _n_softmax(self, n: Node, r):
        x = n.ins[0]
        D = x.base.shape[-1]
        r["dims"][0:2] = (x.base.numel() // D, D)
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)

    _n_logsoftmax = _n_softmax

    def _n_nll(self, n: Node, r):
        x = n.ins[0]
        B, Cc = x.base.shape
        r["dims"][0:2] = (B, Cc)
        r["kind"] = n.attrs["reduction"]
        r["f"][0] = n.attrs["scale"]
        r["aux"][0] = self._const(n.attrs["target"], torch.int64).data_ptr()
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)

    def _n_bce_logits(self, n: Node, r):
        x = n.ins[0]
        r["n"] = x.base.numel()
        r["aux"][0] = self._const(n.attrs["target"], torch.float32).data_ptr()
        self._slot(r, 0, x, x.base)
        self._slot(r, 3, n.out, None)

    def _n_embedding(self, n: Node, r):
        w = n.ins[0]
        idx = n.attrs["indices"]
        V, D = w.base.shape
        pad = n.attrs["padding_idx"]
        r["dims"][0:4] = (idx.numel(), D, V, -1 if pad is None else pad)
        r["aux"][0] = self._const(idx, torch.int64).data_ptr()
        # the token positions stably sorted by table row, then for each sorted position the end of the row's run if
        # one starts there (else 0): the backward adds each row's tokens in a fixed order without atomics
        def runs(src=idx):
            ids, order = torch.sort(src.detach().reshape(-1).to(torch.int64), stable=True)
            n = ids.numel()
            starts = torch.ones(n, dtype=torch.bool, device=ids.device)
            starts[1:] = ids[1:] != ids[:-1]
            first = torch.nonzero(starts).reshape(-1)
            ends = torch.zeros(n, dtype=torch.int64, device=ids.device)
            ends[first] = torch.cat([first[1:], first.new_tensor([n])])
            return torch.cat([order, ends])
        r["aux"][1] = self._const(runs(), torch.int64, recipe=runs).data_ptr()
        if not n.out.base.is_contiguous():
            raise UnsupportedGraph("embedding output must be contiguous")
        self._slot(r, 0, w, w.base)
        self._slot(r, 3, n.out, None)

    # ------------------------------------------------------------------------------------------
    def _on_side(self, fn):
        """Run ``fn(stream_ptr)`` on the plan's side stream (stream capture is illegal on the legacy
        default stream), ordered after / before the caller's current stream."""
        cur = torch.cuda.current_stream(self.dev)
        self.side.wait_stream(cur)
        with torch.cuda.stream(self.side):
            fn(self.side.cuda_stream)
        cur.wait_stream(self.side)

    def run_pass(self, pas: int):
        self._on_side(lambda s: N.call("bb_plan_run", self.handle, pas, s))
        cnt = N.lib().bb_plan_launch_count(self.handle, pas)
        N.launch_counter += cnt
        return cnt

    def __call__(self):
        """hv_arena <- H . d_arena"""
        self._on_side(lambda s: N.call("bb_plan_hvp", self.handle, s))
        self._count_iter(1, 0)

    def _count_iter(self, iters: int, extra_per_iter: int):
        per = N.lib().bb_plan_launch_count(self.handle, PASS_TF) + N.lib().bb_plan_launch_count(self.handle, PASS_TB)
        if extra_per_iter and self.uniform_shift is not None:
            per -= 1            # the K-loops skip the folded c*I node
        self.launches_per_iter = per + extra_per_iter
        N.launch_counter += iters * self.launches_per_iter

    def neumann_loop(self, K: int, alpha: float, v: torch.Tensor, p: torch.Tensor, hv: torch.Tensor):
        assert v.data_ptr() == self.d_arena.data_ptr() and hv.data_ptr() == self.hv_arena.data_ptr()
        self._on_side(lambda s: N.call("bb_plan_neumann_loop", self.handle, K, alpha, v.data_ptr(), p.data_ptr(),
                                       hv.data_ptr(), self.layout.total, int(self.use_graph), s))
        self._count_iter(K, 1)

    def cg_loop(self, K: int, cg_alpha: float, x: torch.Tensor, r: torch.Tensor, p: torch.Tensor, hp: torch.Tensor, ws):
        assert p.data_ptr() == self.d_arena.data_ptr() and hp.data_ptr() == self.hv_arena.data_ptr()
        self._on_side(lambda s: N.call("bb_plan_cg_loop", self.handle, K, cg_alpha, x.data_ptr(), r.data_ptr(),
                                       p.data_ptr(), hp.data_ptr(), self.layout.total, ws.ptr, int(self.use_graph), s))
        self._count_iter(K, 3)

    def mixed_seeds(self, x_arena: torch.Tensor):
        """Native epilogue, first half: one more tangent forward/backward along x (the solve result).  Returns
        [(B, d(g.x)/dB)] for every upper-dependent tensor B of the lower forward; `engine.chain_boundary_seeds`
        pushes them through the upper graph.  Replaces the reference's double backward to lambda
        (neumann.py:44-54, cg.py:58-68)."""
        if x_arena.data_ptr() != self.d_arena.data_ptr():
            self.d_arena.copy_(x_arena)
        self._on_side(lambda s: N.call("bb_plan_hvp_replay" if (self.use_graph and self.serves > 1) else "bb_plan_hvp", self.handle, s))
        self._count_iter(1, 0)
        bases = self.boundary_bases or {}
        return [(bases.get(b.vid, b.base), b.at) for b in self.g.boundaries if b.parent is None and b.at is not None]

    # ---- reuse across calls (engine.py plan cache) ------------------------------------------------------------
    def tape_tensors(self) -> List[torch.Tensor]:
        """Every tape tensor this plan reads through a raw pointer or a recipe: bases of live values, the tensors the
        node descriptors were built from, sources of derived constants."""
        seen, out = set(), []

        def add(t):
            if isinstance(t, torch.Tensor) and id(t) not in seen:
                seen.add(id(t))
                out.append(t)

        for v in self.g.values:
            if (v.needed or v.boundary) and v.param_index is None:
                add(v.base)

        def visit(n):
            for key, val in n.attrs.items():
                if key == "members":
                    for m in val:
                        visit(m)
                elif key == "const_srcs":
                    for t in val:
                        add(t)
                elif key != "const":
                    add(val)
            if n.out is not None:
                add(n.out.base)

        for n in self.g.nodes:
            visit(n)
        return out

    def rebind(self, new_tape) -> bool:
        """Serve a new call whose tape has the same signature (trace.tape_signature): the new forward's values are
        copied INTO the tensors this plan already points at (every descriptor, tensor map and captured graph stays
        valid), derived constants are recomputed, value-dependent refusals re-checked, the packs of K-loop constants
        invalidated and the base-backward pass re-run.  Returns False if some tensor cannot be located (caller then
        builds a fresh plan)."""
        from .trace import op_tensors, tensor_locator

        if self._locator is None:
            self._locator = tensor_locator(self.tape)
        cache: dict = {}

        def new_of(t_old):
            loc = self._locator.get(id(t_old))
            if loc is None:
                return None
            i, k = loc
            lst = cache.get(i)
            if lst is None:
                lst = cache[i] = op_tensors(new_tape.ops[i])
            return lst[k]

        param_ids = {id(p) for p in self.tape.params}
        dsts, srcs = [], []
        done = set()
        for t_old in self.tape_tensors():
            if id(t_old) in param_ids:
                continue
            t_new = new_of(t_old)
            if t_new is None:
                return False
            if t_new.data_ptr() == t_old.data_ptr():
                continue                      # same storage both times (views of parameters, upper parameters)
            key = (t_old.data_ptr(), tuple(t_old.shape), t_old.stride())
            if key in done:
                continue
            done.add(key)
            dsts.append(t_old.detach())
            srcs.append(t_new.detach())
        bases = {}
        for b in self.g.boundaries:
            if b.parent is None:
                t_new = new_of(b.base)
                if t_new is None:
                    return False
                bases[b.vid] = t_new          # the NEW upper graph is what the epilogue must differentiate through
        with torch.no_grad():
            if dsts:
                torch._foreach_copy_(dsts, srcs)
            for const, thunk in self._derived:
                const.copy_(thunk())
        for check, msg in getattr(self.g, "validators", ()):
            if check():
                raise UnsupportedGraph(msg)
        self.boundary_bases = bases
        N.call("bb_plan_invalidate_constants", self.handle)
        self.g.loss.root.a.zero_()
        self.buf(self.g.loss, "a").fill_(1.0)
        self.run_pass(PASS_BB)
        self.serves += 1
        return True

    def profile(self, pas: int) -> np.ndarray:
        ms = np.zeros(len(self.recs), dtype=np.float32)
        self._on_side(lambda s: N.call("bb_plan_profile", self.handle, pas, ms.ctypes.data, s))
        return ms

    # ---- roofline bookkeeping -------------------------------------------------------------------
    def node_bytes(self, i: int, pas: int) -> int:
        """ALGORITHMIC bytes of node ``i`` in pass ``pas``: every operand the rule needs is read once and
        every result written once (DESIGN.md "Algorithmic bytes").  Base tensors count at their own width
        (2 B under bf16 autocast), tangents/adjoints at 4 B."""
        n = self.g.nodes[i]
        if n.op == "diagshift":
            return 12 * sum(p.base.numel() for p in n.ins) if pas == PASS_TB else 0
        if n.op == "convblock2":
            # bytes the fused inner block moves (bf16 padded NHWC everywhere, csrc/convblock2.cu): A = conv-output
            # elements (= input elements), q = pooled elements
            A_, q = n.attrs["Y"].numel(), n.out.base.numel()
            if pas == PASS_TF:      # conv reads t_in, x_in writes t_y | stats reads t_y, y | finalize: gather + pooled arrays
                return int(2 * (2 * A_) + 2 * A_ + 2 * (2 * A_) + 2 * A_ + 7 * q)
            # reduce (pooled) | dense reads t_y, y (+ pooled) writes at_y | dgrad reads at_y, a_y writes at_in | wgrad reads 4 operands
            return int(9 * q + 2 * (2 * A_) + 5 * q + 2 * A_ + 2 * (2 * A_) + 2 * A_ + 4 * (2 * A_))
        if n.op == "convblock":
            # what the fused rule streams: x once, then pooled-size arrays (arg-max code 1 B, xhat* 4 B, dxhat* 4 B,
            # pooled tangent / adjoint-tangent 4 B, masked base adjoint 4 B)
            X, q = n.attrs["X"], n.out.base.numel()
            xb = X.numel() * X.element_size()
            ps = 2 if X.dtype in (torch.bfloat16, torch.float16) else 4       # pooled arrays follow the graph precision
            io = 2 if n.out.tfmt == "nhwc_bf16" else 4                        # pooled tangent / adjoint-tangent
            return int(xb + q * (1 + 2 * ps + io if pas == PASS_TF else 1 + 3 * ps + io))
        out_n = n.out.base.numel()
        total = 0
        uses_base = {"unary": (0,), "mul2": (0, 1), "gemm": (0, 1), "conv2d": (0, 1), "batchnorm": (0,),
                     "layernorm": (0,), "softmax": (0,), "logsoftmax": (0,), "bce_logits": (0,)}.get(n.op, ())
        base_of = {0: n.attrs.get("A", n.attrs.get("X")), 1: n.attrs.get("B", n.attrs.get("W"))}
        for k, v in enumerate(n.ins):
            bt = base_of.get(k) if n.op in ("gemm", "conv2d", "batchnorm", "layernorm") else (v.base if v is not None else None)
            if k in uses_base and bt is not None and (pas != PASS_TF or n.op not in ("softmax", "logsoftmax") or True):
                total += bt.numel() * bt.element_size()
            if v is None:
                continue
            m = v.base.numel()
            if pas == PASS_TF:
                total += 4 * m                       # read t_x
            elif pas == PASS_TB:
                total += 4 * m                       # write at_x
                if n.op in ("unary", "mul2", "gemm", "conv2d", "batchnorm", "layernorm", "softmax", "logsoftmax", "bce_logits"):
                    total += 4 * m                   # read t_x (curvature term)
            else:
                total += 4 * m if v.root.param_index is None else 0
        if pas == PASS_TF:
            total += 4 * out_n
        elif pas == PASS_TB:
            total += 8 * out_n                       # read a_y and at_y
        else:
            total += 4 * out_n
        if n.op == "mulc":
            total += 4 * out_n
        if n.op in ("maxpool2d", "embedding", "nll"):
            idx = n.attrs.get("indices", n.attrs.get("target"))
            total += idx.numel() * 8
        return int(total)

    def roofline(self, hbm_gbs: float, which: str = "measured", reps: int = 3) -> dict:
        """Time every node of the two K-loop passes with CUDA events (eager, on the plan's stream) and
        report the dominant one against the HBM roofline, plus the whole-iteration figure."""
        names = {PASS_TF: "tangent-forward", PASS_TB: "tangent-backward"}
        best = None
        it_ms, it_bytes = 0.0, 0
        rows = []
        for pas in (PASS_TF, PASS_TB):
            ms = np.min(np.stack([self.profile(pas) for _ in range(reps)]), axis=0)
            for i, t in enumerate(ms):
                b = self.node_bytes(i, pas)
                it_ms += float(t)
                it_bytes += b
                rows.append((float(t), b, i, pas))
        rows.sort(reverse=True)
        t, b, i, pas = rows[0]
        n = self.g.nodes[i]
        ach = b / (t * 1e-3) / 1e9 if t > 0 else 0.0
        shp = lambda nd: tuple(nd.out.base.shape) if nd.out is not None else ("params",)
        top = [{"node": f"{self.g.nodes[j].op}{shp(self.g.nodes[j])}:{names[q]}", "ms": round(tt, 4),
                "alg_MB": round(bb_ / 1e6, 3)} for tt, bb_, j, q in rows[:6]]
        return {"bound": "hbm", "kernel": f"{n.op}{shp(n)} {names[pas]} ({n.src})",
                "achieved": ach, "peak": hbm_gbs, "unit": "GB/s", "frac": ach / hbm_gbs, "traffic": None,
                "peak_source": which, "kernel_ms": t, "kernel_alg_bytes": b,
                "iteration": {"alg_bytes": it_bytes, "sum_node_ms": it_ms,
                              "achieved_GBps": it_bytes / (it_ms * 1e-3) / 1e9 if it_ms > 0 else 0.0,
                              "frac": (it_bytes / (it_ms * 1e-3) / 1e9) / hbm_gbs if it_ms > 0 else 0.0},
                "top_nodes": top}

    def describe(self) -> List[str]:
        return [f"{i:4d} {n.op:10s} {n.src:40s} out={tuple(n.out.base.shape) if n.out is not None else None}"
                for i, n in enumerate(self.g.nodes)]

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                N.lib().bb_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
