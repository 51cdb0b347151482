"""Caller-side drop-ins (SURVEY.md §8 f4, betty_b200/callers.py) against the reference's own per-tensor forms:
``Problem.synchronize_params`` (problems/problem.py:599-609) on a world_size-2 gloo group, and
``ImplicitProblem.cache_states`` / ``recover_states`` (problems/implicit_problem.py:67-78) on a module + Adam."""
import copy
import os
import socket
import sys
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _reference_sync(self, params, all_reduce=False):
    """The reference's loop, problems/problem.py:603-609 (used when oracle/_ref is not mirrored)."""
    if self._world_size > 1 and self._strategy not in ["fsdp", "accelerate"]:
        for param in params:
            if not all_reduce:
                dist.broadcast(param.data, 0)
            else:
                param.data.div_(self._world_size)
                dist.all_reduce(param.data, op=dist.ReduceOp.SUM)


def _sync_worker(rank, world, port, out_dir):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from betty_b200 import callers
    from oracle import reference as R

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    ref_sync = _reference_sync
    if R.available():
        R.load()
        from betty.problems.problem import Problem

        ref_sync = Problem.synchronize_params
    torch.manual_seed(10 + rank)
    shapes = [(7, 5), (5,), (3, 3, 3, 2), (1,), (13,), ()]
    mine = [torch.nn.Parameter(torch.randn(s)) for s in shapes]
    mine.append(torch.nn.Parameter(torch.randn(6, 4).t()))                       # strided -> per-tensor path
    mine.append(torch.nn.Parameter(torch.randn(4, dtype=torch.float64)))         # not fp32 -> per-tensor path
    theirs = [torch.nn.Parameter(p.detach().clone(memory_format=torch.preserve_format)) for p in mine]
    me = types.SimpleNamespace(_world_size=world, _strategy="distributed")
    ref = types.SimpleNamespace(_world_size=world, _strategy="distributed")
    res = {}
    for mode in (False, True, False):
        callers.synchronize_params(me, mine, all_reduce=mode)
        ref_sync(ref, theirs, all_reduce=mode)
        res[len(res)] = all(torch.equal(a, b) for a, b in zip(mine, theirs))
        with torch.no_grad():
            for a, b in zip(mine, theirs):       # diverge again before the next mode
                d = torch.randn_like(a)
                a.add_(d)
                b.add_(d)
    same_pack = len(me._bb200_sync_packs) == 1
    torch.save({"ok": res, "same_pack": same_pack, "first": mine[0].detach().clone()}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def test_flat_synchronize_params_matches_reference(tmp_path):
    port = _free_port()
    mp.spawn(_sync_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"r{r}.pt") for r in range(2))
    assert all(r0["ok"].values()) and all(r1["ok"].values())
    assert r0["same_pack"] and r1["same_pack"]


def test_single_process_is_a_no_op():
    from betty_b200 import callers

    p = [torch.nn.Parameter(torch.randn(3))]
    before = p[0].detach().clone()
    callers.synchronize_params(types.SimpleNamespace(_world_size=1, _strategy="default"), p)
    assert torch.equal(p[0], before)


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(6, 8)
        self.bn = torch.nn.BatchNorm1d(8)      # running stats (fp32) + num_batches_tracked (int64)
        self.b = torch.nn.Linear(8, 3)

    def forward(self, x):
        return self.b(torch.relu(self.bn(self.a(x))))


def _steps(net, opt, n, seed):
    g = torch.Generator().manual_seed(seed)
    for _ in range(n):
        x = torch.randn(16, 6, generator=g).to(next(net.parameters()).device)
        opt.zero_grad()
        net(x).square().mean().backward()
        opt.step()


def _state_equal(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and torch.equal(a.cpu(), b.cpu())
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_state_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_state_equal(x, y) for x, y in zip(a, b))
    return a == b


def _roll_back_case(device, warm_steps, opt_name):
    from betty_b200 import callers

    torch.manual_seed(0)
    net_a = _Net().to(device)
    net_b = copy.deepcopy(net_a)
    mk = {"adam": lambda ps: torch.optim.Adam(ps, lr=1e-2), "sgd": lambda ps: torch.optim.SGD(ps, lr=1e-2, momentum=0.9)}
    opt_a, opt_b = mk[opt_name](net_a.parameters()), mk[opt_name](net_b.parameters())
    _steps(net_a, opt_a, warm_steps, 1)
    _steps(net_b, opt_b, warm_steps, 1)
    me = types.SimpleNamespace(module=net_a, optimizer=opt_a)
    callers.cache_states(me)
    # reference implicit_problem.py:67-70
    mod_cache = copy.deepcopy(net_b.state_dict())
    opt_cache = copy.deepcopy(opt_b.state_dict())
    _steps(net_a, opt_a, 3, 2)
    _steps(net_b, opt_b, 3, 2)
    opt_a.param_groups[0]["lr"] = 5.0
    opt_b.param_groups[0]["lr"] = 5.0
    callers.recover_states(me)
    # reference implicit_problem.py:72-78
    net_b.load_state_dict(mod_cache)
    opt_b.load_state_dict(opt_cache)
    assert _state_equal(net_a.state_dict(), net_b.state_dict())
    assert _state_equal(opt_a.state_dict(), opt_b.state_dict())
    assert me.module_state_dict_cache is None and me._bb200_snapshot is None
    # and both continue identically from the restored state
    _steps(net_a, opt_a, 2, 3)
    _steps(net_b, opt_b, 2, 3)
    assert _state_equal(net_a.state_dict(), net_b.state_dict())
    assert _state_equal(opt_a.state_dict(), opt_b.state_dict())


@pytest.mark.parametrize("warm_steps", [0, 2])
@pytest.mark.parametrize("opt_name", ["adam", "sgd"])
def test_arena_snapshot_matches_reference_roll_back(warm_steps, opt_name):
    _roll_back_case("cpu", warm_steps, opt_name)


@pytest.mark.gpu
@pytest.mark.parametrize("warm_steps", [0, 2])
def test_arena_snapshot_on_cuda(warm_steps):
    _roll_back_case("cuda", warm_steps, "adam")


def test_install_callers_rebinds_reference_methods(monkeypatch):
    """The reference's layout (betty/problems/problem.py: Problem.synchronize_params; betty/problems/implicit_problem.py:
    ImplicitProblem.cache_states / recover_states), stood in by empty modules of the same names."""
    from betty_b200 import callers

    Problem = type("Problem", (), {"synchronize_params": lambda self, params, all_reduce=False: None})
    ImplicitProblem = type("ImplicitProblem", (Problem,), {"cache_states": lambda self: None,
                                                            "recover_states": lambda self: None})
    pkg = types.ModuleType("betty_standin")
    mods = {"betty_standin": pkg, "betty_standin.problems": types.ModuleType("betty_standin.problems"),
            "betty_standin.problems.problem": types.SimpleNamespace(Problem=Problem),
            "betty_standin.problems.implicit_problem": types.SimpleNamespace(ImplicitProblem=ImplicitProblem)}
    for name, mod in mods.items():
        monkeypatch.setitem(sys.modules, name, mod)
    callers.install_callers(pkg)
    assert Problem.synchronize_params is callers.synchronize_params
    assert ImplicitProblem.cache_states is callers.cache_states
    assert ImplicitProblem.recover_states is callers.recover_states
