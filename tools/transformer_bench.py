"""The graph transformer (`--model transformer`) against GATv2, GAT and GraphSAGE on one GPU, and its kernels alone.

    python tools/transformer_bench.py [--shape rmat-1m] [--epochs 10] [--rounds 3] [--launches 50]

Workload: 3 layers, hidden 256, 4 heads, bf16, --enable-pipeline, dropout 0.5, on P = 1 (device-timed CUDA-graph
replay) and on a LocalWorld of P = 4 simulated ranks (eager epochs, all ranks on the one GPU).  The four models run in
the same process on the same graph, alternating, so that all see the same clocks.  The kernel section times
pg_tconv_aggregate, pg_tconv_bwd_dst and pg_tconv_bwd_src on the P = 1 graph with a hidden layer's shape (4 heads of
64, bf16) and states their algorithmic bytes (every operand row read or written once) against the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s).  The card's name and power limit are read in the same call.  Prints one JSON object.
"""
import argparse
import gc
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


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def args_for(model, g, n_parts, cuda_graph):
    return argparse.Namespace(model=model, n_heads=4, backend="nccl", dtype="bf16", n_layers=3, n_hidden=256,
                              n_linear=0, n_feat=g.feat.shape[1], n_class=int(g.label.max()) + 1,
                              n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2, weight_decay=0.0,
                              use_pp=False, enable_pipeline=True, feat_corr=False, grad_corr=False, corr_momentum=0.95,
                              seed=0, n_epochs=0, log_every=10, n_partitions=n_parts, cuda_graph=cuda_graph)


def time_replays(eng, epochs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(epochs):
        eng.run_epoch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / epochs


def time_local(tr, epochs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(epochs):
        tr.run_epoch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / epochs


def kernel_times(graph, launches):
    """ms per launch and algorithmic bytes of the three graph-transformer passes at a hidden layer's shape."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    H, D, dt = 4, 64, torch.bfloat16
    n_in, n_all, nnz = graph.num_in, graph.num_all, graph.nnz
    gen = torch.Generator(device="cuda").manual_seed(0)

    def rows(n):
        t = alloc_rows(n, H * D, dt, "cuda")
        t.copy_(torch.randn(n, H * D, generator=gen, device="cuda"))
        return t

    q, skip, g, k, v = rows(n_in), rows(n_in), rows(n_in), rows(n_all), rows(n_all)
    out, m, s = ops.transformer_aggregate(graph, q, k, v, skip, H)
    dq, gc, delta = ops.transformer_bwd_dst(graph, q, k, v, g, m, s, H)
    dk, dv = ops.transformer_bwd_src(graph, q, k, v, g, m, s, delta, H)
    row, stats = H * D * 2, n_in * H * 4
    # index arrays, then every operand row once: k / v (/ dk / dv) [n_all], q / skip / g / out / dq / g copy [n_in],
    # fp32 statistics [n_in, H]
    passes = {
        "tconv_aggregate": (lambda: ops.transformer_aggregate(graph, q, k, v, skip, H),
                            4 * nnz + 4 * (n_in + 1) + 2 * n_all * row + 3 * n_in * row + 2 * stats),
        "tconv_bwd_dst": (lambda: ops.transformer_bwd_dst(graph, q, k, v, g, m, s, H, dq=dq, gc=gc),
                          4 * nnz + 4 * (n_in + 1) + 2 * n_all * row + 4 * n_in * row + 3 * stats),
        "tconv_bwd_src": (lambda: ops.transformer_bwd_src(graph, q, k, v, g, m, s, delta, H, dk=dk, dv=dv),
                          4 * nnz + 4 * (n_all + 1) + 4 * n_all * row + 2 * n_in * row + 3 * stats),
    }
    res = {}
    for name, (fn, nbytes) in passes.items():
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / launches
        res[name] = dict(ms=round(ms, 4), bytes=int(nbytes), gbps=round(nbytes / ms / 1e6, 1),
                         share_of_hbm=round(nbytes / (ms * 1e-3) / HBM_BPS, 3))
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--shape", default="rmat-1m")
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transformer_bench needs a CUDA device")
    torch.cuda.set_device(0)
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer, RankEngine
    from pipegcn_b200.world import LocalWorld
    g = make_graph(a.shape, device="cuda")
    result = dict(card=card(), shape=a.shape, workload="3 layers, hidden 256, 4 heads, bf16, --enable-pipeline, "
                                                      "dropout 0.5")

    # ---- P = 1, CUDA-graph replay, alternating
    lay1 = build_layouts(g, random_partition(g.n_nodes, 1), 1)[0]
    engines = {}
    for model in ("transformer", "gatv2", "gat", "graphsage"):
        eng = RankEngine(lay1, args_for(model, g, 1, True), LocalWorld(1, "cuda").view(0))
        for _ in range(3):
            eng.run_epoch()
        eng.capture()
        engines[model] = eng
    p1 = {m: [] for m in engines}
    for _ in range(a.rounds):
        for m, eng in engines.items():
            p1[m].append(round(time_replays(eng, a.epochs), 3))
    result["p1_ms_per_epoch_graph_replay"] = p1
    result["kernels_hidden_layer_h4_d64_bf16"] = kernel_times(engines["transformer"].graph, a.launches)
    del engines
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()                  # the four P = 4 trainers' symmetric heaps are plain cudaMallocs
    print(json.dumps(result), file=sys.stderr, flush=True)
    from pipegcn_b200 import ops
    ops.STEP_DEV = None                       # the captured engines' device step counter

    # ---- LocalWorld P = 4 on the one GPU, eager epochs, alternating
    lays4 = build_layouts(g, random_partition(g.n_nodes, 4), 4)
    trainers = {m: LocalTrainer(lays4, args_for(m, g, 4, False), LocalWorld(4, "cuda"))
                for m in ("transformer", "gatv2", "gat", "graphsage")}
    for tr in trainers.values():
        for _ in range(2):
            tr.run_epoch()
    p4 = {m: [] for m in trainers}
    for _ in range(a.rounds):
        for m, tr in trainers.items():
            p4[m].append(round(time_local(tr, a.epochs), 3))
    result["localworld_p4_ms_per_epoch_eager"] = p4
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
