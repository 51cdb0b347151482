"""cg_global on a GPU with the native slice kernels (world_size 1 over NCCL: the collectives degenerate, the K2 / K3 slice
calls, the device-side completion of the two scalars and the plan's H.d do not): must equal the `cg` plugin."""
import os
import socket

import pytest
import torch
import torch.distributed as dist

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture
def single_rank_group():
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()))
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1)
    yield
    dist.destroy_process_group()


@pytest.mark.parametrize("factory,kw", [("mlp_reweight", dict(method="cg", K=5)),
                                        ("learning_to_reweight", dict(method="cg", batch=32, K=6)),
                                        ("logistic_regression_hpo", dict(method="cg", K=3, alpha=0.1))])
def test_cg_global_equals_cg_on_one_rank(single_rank_group, factory, kw):
    from betty_b200 import hypergradient as H
    from betty_b200 import workloads as W
    from tests.helpers import rel_l2

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    wl = W.FACTORIES[factory](device="cuda", **kw)
    want = H.cg(wl.vector, wl.lower, wl.upper, False)
    got = H.jvp_fn_mapping["cg_global"](wl.vector, wl.lower, wl.upper, False)
    err = rel_l2(got, want)
    print(f"[cg_global] {factory}: vs cg {err:.3e}")
    assert err < 1e-4, err          # same kernels, same order of operations; only the graph replay differs
    for p in wl.upper.trainable_parameters():
        p.grad = None
    assert H.jvp_fn_mapping["cg_global"](wl.vector, wl.lower, wl.upper, True) is None
    assert rel_l2([p.grad for p in wl.upper.trainable_parameters()], want) < 1e-4


# ---- 2 GPUs over NCCL: the global-batch solve against the single-process reference on the concatenated batch -------
def _batches(world):
    out = []
    for rank in range(world):
        g = torch.Generator().manual_seed(100 + rank)
        out.append((torch.randn(64, 32, generator=g), torch.randint(0, 10, (64,), generator=g)))
    return out


def _worker(rank, world, port, out_dir):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from betty_b200 import hypergradient as H
    from betty_b200 import workloads as W

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    wl = W.mlp_reweight(device=dev, method="cg", K=4, seed=0)         # same parameters on every rank
    x, y = _batches(world)[rank]
    wl.lower.cur_batch = (x.to(dev), y.to(dev))                        # rank-specific lower batch
    g = torch.Generator().manual_seed(7 + rank)                        # rank-specific right-hand side
    vec = [torch.randn(p.shape, generator=g).to(dev) for p in wl.lower.trainable_parameters()]
    got = H.jvp_fn_mapping["cg_global"](vec, wl.lower, wl.upper, False)
    torch.save({"hg": [t.detach().cpu() for t in got], "v": [t.cpu() for t in vec]}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_cg_global_two_ranks_match_the_reference_on_the_concatenated_batch(tmp_path):
    import torch.multiprocessing as mp

    from betty_b200 import workloads as W
    from oracle import ref_port
    from tests.helpers import rel_l2

    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    recs = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    for a, b in zip(recs[0]["hg"], recs[1]["hg"]):
        assert torch.equal(a, b)                                        # one global solution on every rank
    # single process, fp32 on the CPU: loss of the concatenated batch = mean of the per-rank losses
    wl = W.mlp_reweight(device="cpu", method="cg", K=4, seed=0)
    bs = _batches(world)
    wl.lower.cur_batch = (torch.cat([b[0] for b in bs]), torch.cat([b[1] for b in bs]))
    in_grad = ref_port.lower_gradient(wl.lower)
    hvp = ref_port.make_hvp(in_grad, wl.lower.parameters())
    v_mean = [(a + b) / world for a, b in zip(recs[0]["v"], recs[1]["v"])]
    x = ref_port.cg_solve(v_mean, hvp, 4, 1.0)
    want = ref_port.mixed_product(in_grad, wl.upper, x, False)
    err = rel_l2(recs[0]["hg"], want)
    print(f"[cg_global, 2 ranks over NCCL] vs single-process reference on the concatenated batch: {err:.3e}")
    assert err < 1e-4, err
