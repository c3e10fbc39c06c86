"""Residual gated graph convolution (`--model resgatedgcn`) against GraphSAGE-mean and the graph transformer with one
head on one GPU, and the ResGatedGCN kernels alone.

    python tools/resgated_bench.py [--epochs 10] [--rounds 3] [--launches 50] [--workloads rmat-1m,reddit-shaped]

Workloads (--enable-pipeline, dropout 0.5, P = 1, device-timed CUDA-graph replay): rmat-1m with 3 layers of 256 in
bf16, and reddit-shaped with 4 layers of 256 in fp32.  The transformer at --n-heads 1 runs the same paired GEMMs as
ResGatedGCN around a different gather, so the difference between the two is the gather.  The three models run in the
same process on the same graph, alternating round by round, so that all see the same clocks; the growth of the
device's peak allocation while each model is built and run is its memory.  The kernel section times each ResGatedGCN
pass on the P = 1 graph at a hidden layer's shape (d = d_out = 256, the workload's dtype) and states its algorithmic
bytes, computed from shapes, against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card's name, power limit
and max SM clock are read in the same call.  Every workload runs in a process of its own; each leg's JSON line is
printed as it finishes, then one JSON object of all.
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
MODELS = ("resgatedgcn", "graphsage", "transformer")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def args_for(model, g, wl):
    return argparse.Namespace(model=model, backend="nccl", dtype=wl["dtype"], n_layers=wl["n_layers"], n_hidden=256,
                              n_linear=0, n_feat=g.feat.shape[1], n_class=int(g.label.max()) + 1,
                              n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2, weight_decay=0.0,
                              use_pp=False, enable_pipeline=True, feat_corr=False, grad_corr=False,
                              corr_momentum=0.95, seed=0, n_epochs=0, log_every=10, n_partitions=1, cuda_graph=True,
                              n_heads=1)


def timed(fn, epochs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(epochs):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / epochs


def resgated_bytes(graph, d, es):
    """Algorithmic bytes of one launch of each ResGatedGCN pass at d = half = 256, activation element size es.  N =
    inner rows, U = all rows.  Per edge the aggregate and the destination pass read the source's q and val and the
    source pass the destination's k and G; per row the aggregate reads k and skip and writes out, the destination pass
    reads k and G and writes [dk | G], the source pass reads q and val and writes [dq | dval]."""
    n, u, nnz = graph.num_in, graph.num_all, graph.nnz
    return {
        "pg_resgated_aggregate": 4 * nnz + 2 * es * d * nnz + 3 * es * d * n,
        "pg_resgated_bwd_dst": 4 * nnz + 2 * es * d * nnz + 4 * es * d * n,
        "pg_resgated_bwd_src": 4 * nnz + 2 * es * d * nnz + 4 * es * d * u,
    }


def kernel_times(graph, dtype, launches):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    d = 256
    n, u = graph.num_in, graph.num_all
    gen = torch.Generator(device="cuda").manual_seed(0)

    def rnd(rows, cols):
        t = alloc_rows(rows, cols, dtype, "cuda")
        t.copy_(torch.randn(rows, cols, generator=gen, device="cuda"))
        return t

    qv, ks, g = rnd(u, 2 * d), rnd(n, 2 * d), rnd(n, d)
    calls = {
        "pg_resgated_aggregate": lambda: ops.resgated_aggregate(graph, qv, ks, d, d),
        "pg_resgated_bwd_dst": lambda: ops.resgated_bwd_dst(graph, qv, ks, g, d, d),
        "pg_resgated_bwd_src": lambda: ops.resgated_bwd_src(graph, qv, ks, g, d, d),
    }
    nbytes = resgated_bytes(graph, d, qv.element_size())
    res = {}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        ms = timed(fn, launches)
        res[name] = dict(ms=round(ms, 4), bytes=int(nbytes[name]), gbps=round(nbytes[name] / ms / 1e6, 1),
                         bytes_over_time_vs_hbm=round(nbytes[name] / (ms * 1e-3) / HBM_BPS, 3))
    return res


def _built(make):
    """(object, growth of the device's peak allocation in GB while `make` ran)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    obj = make()
    torch.cuda.synchronize()
    return obj, round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)


def bench_leg(shape, a):
    """One workload (a process of its own, so that every leg starts on an empty card)."""
    from pipegcn_b200 import ops
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    wl = WORKLOADS[shape]
    g = make_graph(shape, device="cuda")
    dtype = torch.bfloat16 if wl["dtype"] == "bf16" else torch.float32
    lay = build_layouts(g, random_partition(g.n_nodes, 1), 1)[0]
    engines, mem = {}, {}

    def make(model):
        ops.STEP_DEV = None
        eng = RankEngine(lay, args_for(model, g, wl), LocalWorld(1, "cuda").view(0))
        for _ in range(3):
            eng.run_epoch()
        eng.capture()
        return eng

    for model in MODELS:
        engines[model], mem[model] = _built(lambda: make(model))
    p1 = {m: [] for m in engines}
    for _ in range(a.rounds):
        for m, eng in engines.items():
            p1[m].append(round(timed(eng.run_epoch, a.epochs), 3))
    return {"p1_ms_per_epoch_graph_replay": p1, "p1_peak_alloc_growth_gb": mem,
            "kernels_hidden_layer_d256": kernel_times(engines["resgatedgcn"].graph, dtype, a.launches)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    p.add_argument("--workloads", default="rmat-1m,reddit-shaped")
    p.add_argument("--leg", default=None, help=argparse.SUPPRESS)      # a workload, run in a child process
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resgated_bench needs a CUDA device")
    torch.cuda.set_device(0)
    if a.leg is not None:
        print(json.dumps(bench_leg(a.leg, a)))
        return
    result = dict(card=card())
    print(json.dumps(result), flush=True)
    for shape in a.workloads.split(","):
        wl = WORKLOADS[shape]
        res = dict(workload=f"{wl['n_layers']} layers, hidden 256, {wl['dtype']}, --enable-pipeline, dropout 0.5, "
                            "P = 1, CUDA-graph replay")
        cmd = [sys.executable, __file__, "--leg", shape, "--epochs", str(a.epochs), "--rounds", str(a.rounds),
               "--launches", str(a.launches)]
        run = subprocess.run(cmd, capture_output=True, text=True)
        if run.returncode == 0:
            leg = json.loads(run.stdout.strip().splitlines()[-1])
        else:
            tail = (run.stderr.strip().splitlines() or ["?"])[-1]
            leg = {"p1": f"not measured: {tail[:300]}"}
        res.update(leg)
        print(json.dumps({shape: leg}), flush=True)
        result[shape] = res
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
