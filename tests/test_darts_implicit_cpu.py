"""CPU tests (float64) of the lowering rules the DARTS search cells need under Neumann / CG: depthwise convolutions,
average pooling that excludes the padding, channel concatenation, convolutions of strided views and global average
pooling.  The torch interpreter of the lowered IR must reproduce autograd's double-backward H.v (what the reference
evaluates) on both DARTS networks and on one small net per rule; the native plan's descriptors must build for both
networks, and the cases still outside the kernels' scope must be refused by name."""
import itertools

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from betty_b200 import workloads as W
from betty_b200.arena import ArenaLayout
from betty_b200.ir import UnsupportedGraph, lower_tape
from betty_b200.plan import OPS, HvpPlan
from betty_b200.trace import record_tape
from tests.helpers import rel_l2, to_double
from tests.interp_ext import Interp

NETS = {
    "lite": lambda: W.darts_search(batch=2, c=4, cells=2, method="neumann", l2=0.01),
    "full": lambda: W.darts_search_full(batch=2, c=4, layers=3, method="cg", l2=0.01),
}


def trace_wl(wl):
    params = wl.lower.trainable_parameters()
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    return loss, tape, params


def check_hvp(loss, tape, params, vec, tol=1e-9):
    g = lower_tape(tape)
    it = Interp(g, torch.float64)
    it.base_backward()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    assert rel_l2([p.a for p in g.params], in_grad) < 1e-10
    for v in (vec, [torch.randn_like(p) for p in params]):
        want = torch.autograd.grad(in_grad, params, grad_outputs=v, retain_graph=True)
        got = it.hvp(list(v))
        assert rel_l2(got, want) < tol
    return g


@pytest.mark.parametrize("net", sorted(NETS))
def test_darts_networks_interp_hvp_matches_autograd(net):
    wl = to_double(NETS[net]())
    loss, tape, params = trace_wl(wl)
    g = check_hvp(loss, tape, params, wl.vector)
    convs = [n for n in g.nodes if n.op == "conv2d"]
    assert any(n.attrs["groups"] > 1 for n in convs)
    assert any(n.op == "avgpool2d" and n.attrs.get("exclude_pad") for n in g.nodes)
    if net == "full":
        # both reduction cells (layers // 3 and 2 * layers // 3 of 3 layers) with their halving shortcut
        assert sum(c.reduction for c in wl.lower.module.cells) == 2
        assert any(n.src.endswith("(contiguous input)") for n in g.nodes)


@pytest.mark.parametrize("net", sorted(NETS))
def test_darts_plan_descriptors_build(net):
    wl = NETS[net]()
    loss, tape, params = trace_wl(wl)
    lay = ArenaLayout.like(params)
    plan = HvpPlan(tape, params, lay, lay.new("cpu"), lay.new("cpu"), dry_run=True)
    dw = [r for r, n in zip(plan.recs, plan.g.nodes) if n.op == "conv2d" and n.attrs["groups"] > 1]
    assert dw and all(int(r["dims"][15]) == int(r["dims"][1]) == int(r["dims"][4]) for r in dw)
    pools = [r for r, n in zip(plan.recs, plan.g.nodes) if n.op == "avgpool2d" and n.attrs.get("exclude_pad")]
    assert pools and all(int(r["kind"]) == 1 for r in pools)
    assert set(int(o) for o in plan.recs["op"]) <= set(OPS.values())


# ---- one small net per rule -----------------------------------------------------------------------------------------
def _hvp_small(body, shape=(2, 3, 9, 11), classes=5):
    torch.manual_seed(0)
    stem = nn.Conv2d(shape[1], 6, 3, padding=1).double()
    mods = nn.ModuleList([stem, *body]).double()
    x = torch.randn(*shape, dtype=torch.float64)
    y = torch.randint(0, classes, (shape[0],))
    head = {}

    def fwd():
        h = torch.tanh(stem(x))
        h = mods_forward(h)
        if "lin" not in head:
            head["lin"] = nn.Linear(h.shape[1], classes).double()
            mods.append(head["lin"])
        return F.cross_entropy(head["lin"](h), y)

    def mods_forward(h):
        for m in body:
            h = m(h)
        return h

    fwd()                                              # builds the head
    params = [p for p in mods.parameters()]
    loss, tape = record_tape(fwd, params)
    vec = [torch.randn_like(p) for p in params]
    return check_hvp(loss, tape, params, vec)


class Flat(nn.Module):
    def __init__(self, keepdim=False):
        super().__init__()
        self.keepdim = keepdim

    def forward(self, h):
        if self.keepdim:
            return h.mean((-1, -2), keepdim=True).flatten(1)
        return h.mean((2, 3))


class Tanh(nn.Module):
    def forward(self, h):
        return torch.tanh(h)


@pytest.mark.parametrize("k,dil,stride", list(itertools.product((3, 5), (1, 2), (1, 2))))
def test_depthwise_conv_rule(k, dil, stride):
    body = [nn.Conv2d(6, 6, k, stride=stride, padding=dil * (k - 1) // 2, dilation=dil, groups=6, bias=(k == 5)),
            Tanh(), nn.Conv2d(6, 4, 1), Tanh(), Flat()]
    g = _hvp_small(body)
    assert any(n.op == "conv2d" and n.attrs["groups"] == 6 for n in g.nodes)


@pytest.mark.parametrize("stride", (1, 2))
def test_avg_pool_excluding_padding_rule(stride):
    body = [nn.AvgPool2d(3, stride=stride, padding=1, count_include_pad=False), Tanh(), nn.Conv2d(6, 4, 1), Tanh(),
            Flat()]
    g = _hvp_small(body)
    assert any(n.op == "avgpool2d" and n.attrs["exclude_pad"] for n in g.nodes)


class CatConst(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(6, 3, 1)
        self.register_buffer("c", torch.randn(1, 2, 1, 1))

    def forward(self, h):
        const = self.c.expand(h.shape[0], 2, h.shape[2], h.shape[3])
        return torch.cat([torch.tanh(self.conv(h)), const, h], dim=1)


def test_cat_with_constant_input_rule():
    g = _hvp_small([CatConst(), nn.Conv2d(11, 4, 3, padding=1), Tanh(), Flat()])
    copies = [n for n in g.nodes if n.src == "aten.cat.default"]
    assert len(copies) == 2 and all(n.out.parent is not None for n in copies)


class SliceConv(nn.Module):
    def __init__(self):
        super().__init__()
        self.even = nn.Conv2d(6, 3, 1, stride=2, bias=False)
        self.odd = nn.Conv2d(6, 3, 1, stride=2, bias=False)

    def forward(self, h):
        return torch.cat([self.even(h), self.odd(h[:, :, 1:, 1:])], dim=1)


def test_strided_slice_conv_input_rule():
    g = _hvp_small([SliceConv(), Tanh(), Flat()], shape=(2, 3, 10, 12))
    assert sum(n.src.endswith("(contiguous input)") for n in g.nodes) == 1


@pytest.mark.parametrize("keepdim", (False, True))
def test_global_mean_rule(keepdim):
    g = _hvp_small([nn.Conv2d(6, 4, 3, padding=1), Tanh(), Flat(keepdim)])
    pools = [n for n in g.nodes if n.op == "avgpool2d"]
    assert len(pools) == 1 and pools[0].attrs["kernel"] == (9, 11)


def test_contiguous_conv_input_lowers_to_one_node():
    g = _hvp_small([nn.Conv2d(6, 4, 3, padding=1), Tanh(), Flat()])
    assert [n.op for n in g.nodes if n.op in ("conv2d", "copy")] == ["conv2d", "conv2d"]


# ---- still refused --------------------------------------------------------------------------------------------------
def _plan_of(body, autocast=False, shape=(2, 8, 9, 9)):
    torch.manual_seed(0)
    mods = nn.ModuleList(body)
    x = torch.randn(*shape)
    params = list(mods.parameters())

    def fwd():
        h = x
        for m in body:
            h = m(h)
        return h.float().pow(2).mean()

    if autocast:
        with torch.autocast("cpu", dtype=torch.bfloat16):
            loss, tape = record_tape(fwd, params)
    else:
        loss, tape = record_tape(fwd, params)
    lay = ArenaLayout.like(params)
    return HvpPlan(tape, params, lay, lay.new("cpu"), lay.new("cpu"), dry_run=True)


@pytest.mark.parametrize("body,autocast,match", [
    ([nn.Conv2d(8, 8, 3, padding=1, groups=2)], False, "grouped convolution"),
    ([nn.Conv2d(8, 16, 3, padding=1, groups=8)], False, "channel multiplier 2"),
    ([nn.Conv2d(8, 8, 3, padding=1, groups=8)], True, "bf16 / fp16"),
    ([nn.Conv2d(8, 8, 1), nn.AvgPool2d(3, stride=2, padding=1, ceil_mode=True)], False, "ceil_mode"),
], ids=["groups2", "multiplier2", "bf16", "ceil_mode"])
def test_out_of_scope_cases_are_refused(body, autocast, match):
    with pytest.raises(UnsupportedGraph, match=match):
        _plan_of(body, autocast)


def test_depthwise_grouped_plan_builds():
    plan = _plan_of([nn.Conv2d(8, 8, 3, padding=1, groups=8)])
    assert int(plan.recs["dims"][0][15]) == 8


@pytest.mark.parametrize("net", sorted(NETS))
def test_cached_plan_locates_every_tensor_of_a_new_call(net):
    """A cached plan serves a later call with the same signature by copying the new forward's values behind its
    pointers (HvpPlan.rebind).  Every tensor the plan reads must be located in the new tape -- including the cat slices
    and pooled views of the lowering, which are refreshed through the tape tensor holding them, and the contiguous
    copies of strided conv inputs, which are recomputed from their new source -- and after the copies every value the
    plan reads equals that of a fresh lowering of the new call."""
    from betty_b200.trace import tape_signature, tensor_locator

    wl = NETS[net]()
    _, tape, params = trace_wl(wl)
    lay = ArenaLayout.like(params)
    plan = HvpPlan(tape, params, lay, lay.new("cpu"), lay.new("cpu"), dry_run=True)
    assert (len(plan.g.derived) > 0) == (net == "full")
    g = torch.Generator().manual_seed(5)
    x, y = wl.lower.cur_batch
    wl.lower.cur_batch = (torch.randn(x.shape, generator=g), y.flip(0))
    with torch.no_grad():
        for a in wl.upper.module.parameters():
            a.add_(0.5 * torch.randn(a.shape, generator=g))
    _, tape2, _ = trace_wl(wl)
    assert tape_signature(tape2) == tape_signature(tape)
    got = plan.rebind_copies(tape2)
    assert got is not None
    dsts, srcs, _ = got
    with torch.no_grad():
        torch._foreach_copy_(dsts, srcs)
        for copy, src in plan.g.derived:
            copy.copy_(src)
    fresh = lower_tape(tape2)
    assert len(fresh.values) == len(plan.g.values)
    # what the plan reads: the tape tensors it lists, and the values the lowering itself made (not in the tape)
    reads = {id(t) for t in plan.tape_tensors()}
    located = tensor_locator(tape)
    used = {id(v) for n in plan.g.nodes for v in list(n.ins) + [n.out] if v is not None}
    compared = made = 0
    for vo, vn in zip(plan.g.values, fresh.values):
        lowering_made = id(vo.base) not in located and (vo.needed or id(vo) in used)
        made += lowering_made
        if vo.param_index is None and (id(vo.base) in reads or lowering_made):
            assert torch.equal(vo.base, vn.base), (net, vo)
            compared += 1
    assert compared > 50 and (made > 0) == (net == "full")
