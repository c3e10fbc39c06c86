"""GraphConv (`--model graphconv`) against GraphSAGE on one GPU, and the scaled gather against the plain one.

    python tools/graphconv_bench.py [--epochs 10] [--rounds 3] [--launches 50] [--workloads rmat-1m,reddit-shaped]

Workloads (hidden 256, --enable-pipeline, dropout 0.5): rmat-1m with 3 layers in bf16, at P = 1 (device-timed CUDA-graph
replay) and on a LocalWorld of P = 4 simulated ranks (eager epochs, all ranks on the one GPU); reddit-shaped with 4
layers in fp32 at P = 1 (replay).  The two models run in the same process on the same graph, alternating, so that both
see the same clocks.  The kernel section times pg_aggregate_scaled and pg_aggregate (with a row divisor) per launch at
the hidden layer's shape (256 columns of bf16) over the rmat-1m forward CSR and backward CSC, CUDA events around 50
launches each, and states their algorithmic bytes against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The
card's name, power limit and maximum SM clock are read in the same call.  Prints one JSON object.
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
MODELS = ("graphconv", "graphsage")
WORKLOADS = {"rmat-1m": dict(n_layers=3, dtype="bf16", p4=True), "reddit-shaped": dict(n_layers=4, dtype="fp32", p4=False)}


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def args_for(model, g, n_parts, cuda_graph, n_layers, dtype):
    return argparse.Namespace(model=model, backend="nccl", dtype=dtype, n_layers=n_layers, n_hidden=256, n_linear=0,
                              n_feat=g.feat.shape[1], n_class=int(g.label.max()) + 1,
                              n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2, weight_decay=0.0,
                              use_pp=False, enable_pipeline=True, feat_corr=False, grad_corr=False, corr_momentum=0.95,
                              seed=0, n_epochs=0, log_every=10, n_partitions=n_parts, cuda_graph=cuda_graph)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_times(graph, launches):
    """ms per launch and algorithmic bytes of the scaled and the plain gather, CSR and CSC, 256 bf16 columns."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    d, dt = 256, torch.bfloat16
    gen = torch.Generator(device="cuda").manual_seed(0)
    c = ops.sym_norm(torch.clamp(graph.bwd.indptr[1:] - graph.bwd.indptr[:-1], min=1))
    res = {}
    for direction, plan, n_src in (("csr", graph.fwd, graph.num_all), ("csc", graph.bwd, graph.num_in)):
        x = alloc_rows(n_src, d, dt, "cuda")
        x.copy_(torch.randn(n_src, d, generator=gen, device="cuda"))
        deg = torch.clamp(plan.indptr[1:] - plan.indptr[:-1], min=1).float().contiguous()
        base = 4 * plan.nnz + 4 * (plan.n_rows + 1) + 2 * d * (n_src + plan.n_rows)
        passes = {"aggregate_scaled": (lambda: ops.aggregate_scaled(plan, x, c, c), base + 4 * n_src + 4 * plan.n_rows),
                  "aggregate_row_div": (lambda: ops.aggregate(plan, x, row_div=deg), base + 4 * plan.n_rows)}
        for _ in range(3):
            for fn, _ in passes.values():
                fn()
        for name, (fn, nbytes) in passes.items():
            ms = timed(fn, launches)
            res[f"{direction}_{name}"] = dict(ms=round(ms, 4), bytes=int(nbytes), gbps=round(nbytes / ms / 1e6, 1),
                                              share_of_hbm=round(nbytes / (ms * 1e-3) / HBM_BPS, 3))
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    p.add_argument("--workloads", default="rmat-1m,reddit-shaped")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graphconv_bench needs a CUDA device")
    torch.cuda.set_device(0)
    from pipegcn_b200 import ops
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer, RankEngine
    from pipegcn_b200.world import LocalWorld
    result = dict(card=card(), workload="hidden 256, --enable-pipeline, dropout 0.5")
    for shape in a.workloads.split(","):
        w = WORKLOADS[shape]
        g = make_graph(shape, device="cuda")
        res = dict(n_layers=w["n_layers"], dtype=w["dtype"])
        lay1 = build_layouts(g, random_partition(g.n_nodes, 1), 1)[0]
        engines = {}
        for model in MODELS:
            eng = RankEngine(lay1, args_for(model, g, 1, True, w["n_layers"], w["dtype"]), LocalWorld(1, "cuda").view(0))
            for _ in range(3):
                eng.run_epoch()
            eng.capture()
            engines[model] = eng
        p1 = {m: [] for m in engines}
        for _ in range(a.rounds):
            for m, eng in engines.items():
                p1[m].append(round(timed(eng.run_epoch, a.epochs), 3))
        res["p1_ms_per_epoch_graph_replay"] = p1
        if shape == "rmat-1m":
            result["kernels_hidden_layer_d256_bf16"] = kernel_times(engines["graphconv"].graph, a.launches)
        del engines
        torch.cuda.synchronize()
        ops.STEP_DEV = None                       # the captured engines' device step counter
        if w["p4"]:
            lays4 = build_layouts(g, random_partition(g.n_nodes, 4), 4)
            trainers = {m: LocalTrainer(lays4, args_for(m, g, 4, False, w["n_layers"], w["dtype"]), LocalWorld(4, "cuda"))
                        for m in MODELS}
            for tr in trainers.values():
                for _ in range(2):
                    tr.run_epoch()
            p4 = {m: [] for m in trainers}
            for _ in range(a.rounds):
                for m, tr in trainers.items():
                    p4[m].append(round(timed(tr.run_epoch, a.epochs), 3))
            res["localworld_p4_ms_per_epoch_eager"] = p4
            del trainers
        torch.cuda.synchronize()
        result[shape] = res
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
