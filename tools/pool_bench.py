"""Max-pool GraphSAGE (`--aggregator pool`) against the mean aggregator on one GPU, and the pool kernels alone.

    python tools/pool_bench.py [--epochs 10] [--rounds 3] [--launches 50] [--workloads rmat-1m,reddit-shaped]

Workloads (--enable-pipeline, dropout 0.5): rmat-1m with 3 layers of 256 in bf16, and reddit-shaped with 4 layers of
256 in fp32.  Each runs on P = 1 (device-timed CUDA-graph replay) and on a LocalWorld of P = 4 simulated ranks (eager
epochs, all ranks on the one GPU).  Pool and mean run in the same process on the same graph, alternating, so that
both see the same clocks.  The kernel section times pg_max_aggregate and pg_max_aggregate_bwd on the P = 1 graph at a
hidden layer's shape (d = 256, the workload's dtype) and states their algorithmic bytes against the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s).  The card's name, power limit and max SM clock are read in the same call.
Every workload and partition count runs in a process of its own.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

HBM_BPS = 3.35e12
WORKLOADS = {"rmat-1m": dict(n_layers=3, dtype="bf16"), "reddit-shaped": dict(n_layers=4, dtype="fp32")}


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def args_for(aggregator, g, wl, n_parts, cuda_graph):
    return argparse.Namespace(model="graphsage", aggregator=aggregator, backend="nccl", dtype=wl["dtype"],
                              n_layers=wl["n_layers"], n_hidden=256, n_linear=0, n_feat=g.feat.shape[1],
                              n_class=int(g.label.max()) + 1, n_train=int(g.train_mask.sum()), dropout=0.5,
                              norm="layer", lr=1e-2, weight_decay=0.0, use_pp=False, enable_pipeline=True,
                              feat_corr=False, grad_corr=False, corr_momentum=0.95, seed=0, n_epochs=0, log_every=10,
                              n_partitions=n_parts, cuda_graph=cuda_graph)


def timed(fn, epochs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(epochs):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / epochs


def pool_bytes(graph, d, es):
    """Algorithmic bytes of one launch: the forward reads the column ids and row pointers, gathers s*d per edge and
    writes hn (s*d) and A (4*d) per row; the backward reads the CSC ids and pointers, Q once per source row, A and
    g_neigh (4 + s)*d per edge, and writes gQ (s*d) per source row."""
    n_in, n_all, nnz = graph.num_in, graph.num_all, graph.nnz
    fwd = 4 * nnz + 4 * (n_in + 1) + es * d * nnz + (es + 4) * d * n_in
    bwd = 4 * nnz + 4 * (n_all + 1) + es * d * n_all + (4 + es) * d * nnz + es * d * n_all
    return fwd, bwd


def kernel_times(graph, dtype, launches):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    d = 256
    gen = torch.Generator(device="cuda").manual_seed(0)
    q = alloc_rows(graph.num_all, d, dtype, "cuda")
    q.copy_(torch.randn(graph.num_all, d, generator=gen, device="cuda"))
    gn = alloc_rows(graph.num_in, d, dtype, "cuda")
    gn.copy_(torch.randn(graph.num_in, d, generator=gen, device="cuda"))
    hn, arg = ops.max_aggregate(graph.fwd, q)
    fb, bb = pool_bytes(graph, d, q.element_size())
    res = {}
    for name, fn, nbytes in (("pg_max_aggregate", lambda: ops.max_aggregate(graph.fwd, q), fb),
                             ("pg_max_aggregate_bwd", lambda: ops.max_aggregate_bwd(graph.bwd, q, arg, gn), bb)):
        for _ in range(3):
            fn()
        ms = timed(fn, launches)
        res[name] = dict(ms=round(ms, 4), bytes=int(nbytes), gbps=round(nbytes / ms / 1e6, 1),
                         share_of_hbm=round(nbytes / (ms * 1e-3) / HBM_BPS, 3))
    return res


def bench_leg(shape, n_parts, a):
    """One workload at one partition count (a process of its own, so that every leg starts on an empty card)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer, RankEngine
    from pipegcn_b200.world import LocalWorld
    wl = WORKLOADS[shape]
    g = make_graph(shape, device="cuda")
    dtype = torch.bfloat16 if wl["dtype"] == "bf16" else torch.float32
    out = {}
    if n_parts == 1:        # CUDA-graph replay, alternating
        lay1 = build_layouts(g, random_partition(g.n_nodes, 1), 1)[0]
        engines = {}
        for agg in ("pool", "mean"):
            ops.STEP_DEV = None
            eng = RankEngine(lay1, args_for(agg, g, wl, 1, True), LocalWorld(1, "cuda").view(0))
            for _ in range(3):
                eng.run_epoch()
            eng.capture()
            engines[agg] = eng
        p1 = {m: [] for m in engines}
        for _ in range(a.rounds):
            for m, eng in engines.items():
                p1[m].append(round(timed(eng.run_epoch, a.epochs), 3))
        out["p1_ms_per_epoch_graph_replay"] = p1
        out["kernels_hidden_layer_d256"] = kernel_times(engines["pool"].graph, dtype, a.launches)
        return out
    # LocalWorld of n_parts simulated ranks on the one GPU, eager epochs, alternating
    lays = build_layouts(g, random_partition(g.n_nodes, n_parts), n_parts)
    trainers = {m: LocalTrainer(lays, args_for(m, g, wl, n_parts, False), LocalWorld(n_parts, "cuda"))
                for m in ("pool", "mean")}
    for tr in trainers.values():
        for _ in range(2):
            tr.run_epoch()
    pn = {m: [] for m in trainers}
    for _ in range(a.rounds):
        for m, tr in trainers.items():
            pn[m].append(round(timed(tr.run_epoch, a.epochs), 3))
    out[f"localworld_p{n_parts}_ms_per_epoch_eager"] = pn
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    p.add_argument("--workloads", default="rmat-1m,reddit-shaped")
    p.add_argument("--leg", default=None, help=argparse.SUPPRESS)      # shape:P, run in a child process
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pool_bench needs a CUDA device")
    torch.cuda.set_device(0)
    if a.leg is not None:
        shape, n_parts = a.leg.split(":")
        print(json.dumps(bench_leg(shape, int(n_parts), a)))
        return
    result = dict(card=card())
    for shape in a.workloads.split(","):
        wl = WORKLOADS[shape]
        res = dict(workload=f"{wl['n_layers']} layers, hidden 256, {wl['dtype']}, --enable-pipeline, dropout 0.5")
        for n_parts in (1, 4):
            cmd = [sys.executable, __file__, "--leg", f"{shape}:{n_parts}", "--epochs", str(a.epochs), "--rounds",
                   str(a.rounds), "--launches", str(a.launches)]
            run = subprocess.run(cmd, capture_output=True, text=True)
            if run.returncode == 0:
                res.update(json.loads(run.stdout.strip().splitlines()[-1]))
            else:
                tail = (run.stderr.strip().splitlines() or ["?"])[-1]
                res[f"p{n_parts}"] = f"not measured: {tail[:300]}"
        result[shape] = res
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
