"""world_size-2 gloo tests on the host: the N>1 logic that does not need a GPU.

* the oracle over a real gloo process group (one process per partition, tagged isend/recv like
  PipeGCN/helper/feature_buffer.py:173,179) equals the oracle over the in-process thread fabric;
* `Reducer` (pack -> /n_train -> all-reduce -> unpack) across two processes reproduces the reduced gradients the
  reference's reducer produced (golden fixture);
* `DistWorld.publish/collect` exchanges the per-rank buffer tables.
"""
import os
import socket
import tempfile

import pytest
import torch
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _oracle_worker(rank, size, port, mode_kw, out_dir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=size)
    torch.set_num_threads(1)
    from oracle.fabric import GlooFabric
    from oracle.train import initial_state, run_rank
    from tests.helpers import make_args, small_world
    g, _, _, setups = small_world("tiny", size)
    oargs, _ = make_args(g, 5, n_epochs=3, **mode_kw)
    fab = GlooFabric()
    tr = run_rank(setups[rank], oargs, fab, init_state=initial_state(oargs))
    torch.save({"losses": tr.losses, "logits": tr.logits, "grads": tr.grads}, f"{out_dir}/r{rank}.pt")
    dist.barrier()
    # with --enable-pipeline the messages of the last epoch are never consumed (the reference leaves its transfer
    # threads behind the same way): do not wait for those sends, leave without tearing the group down
    os._exit(0)


@pytest.mark.parametrize("mode_kw", [dict(), dict(enable_pipeline=True, feat_corr=True, grad_corr=True)])
def test_oracle_over_gloo_equals_thread_fabric(mode_kw):
    from oracle.train import initial_state, run_world
    from tests.helpers import make_args, small_world
    size = 2
    out_dir = tempfile.mkdtemp(prefix="pg_gloo_")
    mp.spawn(_oracle_worker, args=(size, _free_port(), mode_kw, out_dir), nprocs=size, join=True)
    g, _, _, setups = small_world("tiny", size)
    oargs, _ = make_args(g, 5, n_epochs=3, **mode_kw)
    ref = run_world(setups, oargs, init_state=initial_state(oargs))
    for r in range(size):
        got = torch.load(f"{out_dir}/r{r}.pt", weights_only=False)
        for e in range(3):
            assert abs(got["losses"][e] - ref[r].losses[e]) <= 1e-5 * abs(ref[r].losses[e])
            torch.testing.assert_close(got["logits"][e], ref[r].logits[e], rtol=1e-5, atol=1e-6)
            for n, t in ref[r].grads[e].items():
                torch.testing.assert_close(got["grads"][e][n], t, rtol=1e-4, atol=1e-7)


def _reducer_worker(rank, size, port, out_dir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=size)
    from pipegcn_b200.helper.reducer import Reducer
    from pipegcn_b200.world import DistWorld
    world = DistWorld(device="cpu")
    world.publish("table", {"rank": rank, "off": [rank * 10, rank * 10 + 1]})
    tables = world.collect("table")
    assert [t["rank"] for t in tables] == list(range(size))
    torch.manual_seed(0)
    model = torch.nn.Linear(7, 3)
    red = Reducer(world)
    red.init(model, world)
    n_train = 11
    for i, (name, p) in enumerate(model.named_parameters()):
        g = torch.full_like(p, float(rank + 1 + i))
        p.grad = g.clone()
        red.reduce(p, name, g, n_train)
    red.synchronize()
    torch.save({n: p.grad.clone() for n, p in model.named_parameters()}, f"{out_dir}/red{rank}.pt")
    dist.barrier()
    dist.destroy_process_group()


def test_reducer_and_world_tables_over_gloo():
    size = 2
    out_dir = tempfile.mkdtemp(prefix="pg_gloo_")
    mp.spawn(_reducer_worker, args=(size, _free_port(), out_dir), nprocs=size, join=True)
    for r in range(size):
        got = torch.load(f"{out_dir}/red{r}.pt", weights_only=False)
        for i, (n, t) in enumerate(got.items()):
            want = sum(float(k + 1 + i) for k in range(size)) / 11          # sum over ranks of grad / n_train
            assert torch.allclose(t, torch.full_like(t, want), rtol=1e-6), (n, t.flatten()[0].item(), want)


def test_metis_partition_is_valid_and_balanced():
    from pipegcn_b200.metis import metis_partition
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph
    g = make_graph("tiny")
    for obj in ("vol", "cut"):
        part = metis_partition(g, 3, obj)
        assert part.shape == (g.n_nodes,) and int(part.min()) == 0 and int(part.max()) == 2
        sizes = torch.bincount(part, minlength=3)
        assert sizes.max().item() <= 1.2 * g.n_nodes / 3 + 2
        lays = build_layouts(g, part, 3)
        assert sum(l.num_in for l in lays) == g.n_nodes
        assert sum(l.nnz for l in lays) == g.n_edges


def _syncbn_worker(rank, size, port, out_dir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=size)
    from pipegcn_b200.module.sync_bn import SyncBatchNorm
    torch.manual_seed(0)
    x_all = torch.randn(40, 6) * 2 + 1
    g_all = torch.randn(40, 6)
    rows = slice(0, 17) if rank == 0 else slice(17, 40)
    bn = SyncBatchNorm(6, whole_size=40)
    with torch.no_grad():
        bn.weight.copy_(torch.linspace(0.5, 1.5, 6))
        bn.bias.copy_(torch.linspace(-1, 1, 6))
    x = x_all[rows].clone().requires_grad_(True)
    y = bn(x)
    y.backward(g_all[rows])
    torch.save({"y": y.detach(), "dx": x.grad, "dw": bn.weight.grad, "db": bn.bias.grad,
                "rm": bn.running_mean.clone(), "rv": bn.running_var.clone()}, f"{out_dir}/bn{rank}.pt")
    dist.barrier()
    dist.destroy_process_group()


def test_sync_batch_norm_equals_batch_norm_on_all_rows():
    """--norm batch (module/sync_bn.py): two partitions with synchronised statistics == BatchNorm1d over all rows
    (biased variance, momentum update of the running statistics with the biased variance as the reference does)."""
    size = 2
    out_dir = tempfile.mkdtemp(prefix="pg_gloo_")
    mp.spawn(_syncbn_worker, args=(size, _free_port(), out_dir), nprocs=size, join=True)
    torch.manual_seed(0)
    x_all = (torch.randn(40, 6) * 2 + 1).requires_grad_(True)
    g_all = torch.randn(40, 6)
    w = torch.linspace(0.5, 1.5, 6).requires_grad_(True)
    b = torch.linspace(-1, 1, 6).requires_grad_(True)
    mean, var = x_all.mean(0), x_all.var(0, unbiased=False)
    y = (x_all - mean) / torch.sqrt(var + 1e-5) * w + b
    y.backward(g_all)
    got = [torch.load(f"{out_dir}/bn{r}.pt", weights_only=False) for r in range(size)]
    torch.testing.assert_close(torch.cat([got[0]["y"], got[1]["y"]]), y.detach(), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(torch.cat([got[0]["dx"], got[1]["dx"]]), x_all.grad, rtol=1e-4, atol=1e-5)
    for r in range(size):            # parameter gradients are already summed over ranks (sync_bn.py:35-36)
        torch.testing.assert_close(got[r]["dw"], w.grad, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(got[r]["db"], b.grad, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(got[r]["rm"], 0.1 * mean.detach(), rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(got[r]["rv"], 0.9 + 0.1 * var.detach(), rtol=1e-4, atol=1e-6)
