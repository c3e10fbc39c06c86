"""GCNII (`--model gcnii`) against GraphConv at equal depth on one GPU, and the residual gather against the scaled one.

    python tools/gcnii_bench.py [--epochs 10] [--rounds 3] [--launches 50] [--depths 4] [--no-p4] [--out FILE]

Workload: rmat-1m, hidden 256, bf16, --enable-pipeline, dropout 0.5.  For every depth (--n-layers; GCNII uses
--n-linear 1, so depth 4 is fc_in + 3 convolutions + a linear, GraphConv 4 graph layers) the two models run in the
same process on the same graph, alternating, so that both see the same clocks: at P = 1 as device-timed CUDA-graph
replay, and on a LocalWorld of P = 4 simulated ranks (eager epochs, all ranks on the one GPU).  Every P = 1 engine's
peak device memory above what was allocated before it is reported.  The kernel section times pg_aggregate_scaled_res
and pg_aggregate_scaled per launch at the hidden layer's shape (256 columns of bf16) over the rmat-1m forward CSR, CUDA events around `--launches`
launches each, with their algorithmic bytes against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card's
name, power limit and maximum SM clock are read in the same call.  Prints one JSON object (and writes it to --out).
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
MODELS = ("gcnii", "graphconv")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def args_for(model, g, n_parts, cuda_graph, n_layers):
    return argparse.Namespace(model=model, backend="nccl", dtype="bf16", n_layers=n_layers, n_hidden=256,
                              n_linear=1 if model == "gcnii" else 0, n_feat=g.feat.shape[1],
                              n_class=int(g.label.max()) + 1, n_train=int(g.train_mask.sum()), dropout=0.5,
                              norm="layer", lr=1e-2, weight_decay=0.0, use_pp=False, enable_pipeline=True,
                              feat_corr=False, grad_corr=False, corr_momentum=0.95, seed=0, n_epochs=0, log_every=10,
                              n_partitions=n_parts, cuda_graph=cuda_graph)


def free():
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


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
    """ms per launch and algorithmic bytes of the residual and the scaled gather over the CSR, 256 bf16 columns."""
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    d, dt = 256, torch.bfloat16
    gen = torch.Generator(device="cuda").manual_seed(0)
    plan, n_src = graph.fwd, graph.num_all
    c = ops.sym_norm(torch.clamp(graph.bwd.indptr[1:] - graph.bwd.indptr[:-1], min=1))
    x = alloc_rows(n_src, d, dt, "cuda")
    x.copy_(torch.randn(n_src, d, generator=gen, device="cuda"))
    h0 = alloc_rows(plan.n_rows, d, dt, "cuda")
    h0.copy_(torch.randn(plan.n_rows, d, generator=gen, device="cuda"))
    cs = (0.9 * c[:plan.n_rows]).contiguous()
    base = 4 * plan.nnz + 4 * (plan.n_rows + 1) + 2 * d * (n_src + plan.n_rows) + 4 * n_src + 4 * plan.n_rows
    passes = {"aggregate_scaled_res": (lambda: ops.aggregate_scaled_res(plan, x, c, cs, res=h0, alpha=0.1),
                                       base + 2 * d * plan.n_rows),
              "aggregate_scaled": (lambda: ops.aggregate_scaled(plan, x, c, cs), base)}
    for _ in range(3):
        for fn, _ in passes.values():
            fn()
    res = {}
    for _ in range(2):                      # alternate, keep the second round
        for name, (fn, nbytes) in passes.items():
            ms = timed(fn, launches)
            res[f"csr_{name}"] = dict(ms=round(ms, 4), bytes=int(nbytes), gbps=round(nbytes / ms / 1e6, 1),
                                      share_of_hbm=round(nbytes / (ms * 1e-3) / HBM_BPS, 3))
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    p.add_argument("--depths", default="4")
    p.add_argument("--no-p4", action="store_true")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gcnii_bench needs a CUDA device")
    torch.cuda.set_device(0)
    from pipegcn_b200 import ops
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer, RankEngine
    from pipegcn_b200.world import LocalWorld
    result = dict(card=card(), workload="rmat-1m, hidden 256, bf16, --enable-pipeline, dropout 0.5")
    g = make_graph("rmat-1m", device="cuda")
    lay1 = build_layouts(g, random_partition(g.n_nodes, 1), 1)[0]
    for depth in [int(s) for s in a.depths.split(",")]:
        res = {}
        engines, mem = {}, {}
        for model in MODELS:
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            eng = RankEngine(lay1, args_for(model, g, 1, True, depth), LocalWorld(1, "cuda").view(0))
            for _ in range(3):
                eng.run_epoch()
            eng.capture()
            eng.run_epoch()
            torch.cuda.synchronize()
            mem[model] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)     # this engine's peak
            engines[model] = eng
        p1 = {m: [] for m in engines}
        for _ in range(a.rounds):
            for m, eng in engines.items():
                p1[m].append(round(timed(eng.run_epoch, a.epochs), 3))
        res["p1_ms_per_epoch_graph_replay"] = p1
        res["p1_peak_device_memory_gib"] = mem
        if "kernels_hidden_layer_d256_bf16" not in result:
            result["kernels_hidden_layer_d256_bf16"] = kernel_times(engines["gcnii"].graph, a.launches)
        del engines, eng
        free()
        ops.STEP_DEV = None                       # the captured engines' device step counter
        if not a.no_p4:
            lays4 = build_layouts(g, random_partition(g.n_nodes, 4), 4)
            trainers = {m: LocalTrainer(lays4, args_for(m, g, 4, False, depth), LocalWorld(4, "cuda")) for m in MODELS}
            for tr in trainers.values():
                for _ in range(2):
                    tr.run_epoch()
            p4 = {m: [] for m in trainers}
            for _ in range(a.rounds):
                for m, tr in trainers.items():
                    p4[m].append(round(timed(tr.run_epoch, a.epochs), 3))
            res["localworld_p4_ms_per_epoch_eager"] = p4
            del trainers, tr
        free()
        result[f"depth{depth}"] = res
        print(json.dumps({f"depth{depth}": res}), file=sys.stderr, flush=True)      # progress
    result["card_after"] = card()
    text = json.dumps(result)
    print(text)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
