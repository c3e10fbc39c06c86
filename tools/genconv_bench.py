"""Softmax-aggregation graph convolution (`--model genconv`, learnt t) against GraphSAGE-mean on one GPU, and the
GENConv kernels alone.

    python tools/genconv_bench.py [--epochs 10] [--rounds 3] [--launches 50] [--workloads rmat-1m,reddit-shaped]

Workloads (--enable-pipeline, dropout 0.5): rmat-1m with 3 layers of 256 in bf16, and reddit-shaped with 4 layers of
256 in fp32.  Each runs on P = 1 (device-timed CUDA-graph replay) and on a LocalWorld of P = 4 simulated ranks (eager
epochs, all ranks on the one GPU).  GENConv and mean run in the same process on the same graph, alternating, so that both
see the same clocks; the growth of the device's peak allocation while each model is built and run is its memory.  The
kernel section times every GENConv kernel on the P = 1 graph at a hidden layer's shape (d = d_out = 256, the workload's
dtype) and states its algorithmic bytes, computed from shapes, against the H100 SXM data-sheet HBM3 bandwidth
(3.35 TB/s).  The card's name, power limit and max SM clock are read in the same call.  Every workload and partition
count runs in a process of its own; each leg's JSON line is printed as it finishes, then one JSON object of all.
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
MODELS = ("genconv", "graphsage")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def args_for(model, g, wl, n_parts, cuda_graph):
    return argparse.Namespace(model=model, backend="nccl", dtype=wl["dtype"], n_layers=wl["n_layers"], n_hidden=256,
                              n_linear=0, n_feat=g.feat.shape[1], n_class=int(g.label.max()) + 1,
                              n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2, weight_decay=0.0,
                              use_pp=False, enable_pipeline=True, feat_corr=False, grad_corr=False,
                              corr_momentum=0.95, seed=0, n_epochs=0, log_every=10, n_partitions=n_parts,
                              cuda_graph=cuda_graph, **(dict(genconv_t=1.0, genconv_learn_t=True)
                                                         if model == "genconv" else {}))


def timed(fn, epochs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(epochs):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / epochs


def genconv_bytes(graph, d, es):
    """Algorithmic bytes of one launch of each GENConv kernel at d = 256 with learnt t, activation element size es.
    N = inner rows, U = all rows.  The aggregate reads one x_src row per edge and writes S, agg, L and var; the source
    pass reads L, G and Q (fp32) of the destination per edge and x_src twice per row (the messages, the ReLU gate)."""
    n, u, nnz = graph.num_in, graph.num_all, graph.nnz
    return {
        "pg_genconv_aggregate": 4 * nnz + es * d * nnz + 2 * es * d * n + 12 * d * n,
        "pg_genconv_bwd_dst": 16 * d * n + (es * d * n if es == 2 else 0),
        "pg_genconv_bwd_src": 4 * nnz + 12 * d * nnz + 3 * es * d * u,
    }


def kernel_times(graph, dtype, launches):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    d = 256
    n, u = graph.num_in, graph.num_all
    gen = torch.Generator(device="cuda").manual_seed(0)

    def rnd(rows, cols, dt):
        t = alloc_rows(rows, cols, dt, "cuda")
        t.copy_(torch.randn(rows, cols, generator=gen, device="cuda"))
        return t

    xs, xd, gs = rnd(u, d, dtype), rnd(n, d, dtype), rnd(n, d, torch.float32)
    t = torch.ones(1, device="cuda")
    s, agg, lse, var = ops.genconv_aggregate(graph.fwd, xs, xd, t, None, n, stats=True, learn_t=True)
    gdt = dtype if dtype != torch.float32 else None
    q, _, _ = ops.genconv_bwd_dst(gs, agg, t, var, dtype=gdt)
    calls = {
        "pg_genconv_aggregate": lambda: ops.genconv_aggregate(graph.fwd, xs, xd, t, None, n, stats=True, learn_t=True),
        "pg_genconv_bwd_dst": lambda: ops.genconv_bwd_dst(gs, agg, t, var, dtype=gdt),
        "pg_genconv_bwd_src": lambda: ops.genconv_bwd_src(graph.bwd, xs, t, lse, gs, q, None, n),
    }
    nbytes = genconv_bytes(graph, d, xs.element_size())
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
        engines, mem = {}, {}

        def make(model):
            ops.STEP_DEV = None
            eng = RankEngine(lay1, args_for(model, g, wl, 1, True), LocalWorld(1, "cuda").view(0))
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
        out["p1_ms_per_epoch_graph_replay"] = p1
        out["p1_peak_alloc_growth_gb"] = mem
        out["kernels_hidden_layer_d256"] = kernel_times(engines["genconv"].graph, dtype, a.launches)
        return out
    # LocalWorld of n_parts simulated ranks on the one GPU, eager epochs, alternating
    lays = build_layouts(g, random_partition(g.n_nodes, n_parts), n_parts)
    trainers, mem = {}, {}

    def make_tr(model):
        tr = LocalTrainer(lays, args_for(model, g, wl, n_parts, False), LocalWorld(n_parts, "cuda"))
        for _ in range(2):
            tr.run_epoch()
        return tr

    for model in MODELS:
        trainers[model], mem[model] = _built(lambda: make_tr(model))
    pn = {m: [] for m in trainers}
    for _ in range(a.rounds):
        for m, tr in trainers.items():
            pn[m].append(round(timed(tr.run_epoch, a.epochs), 3))
    out[f"localworld_p{n_parts}_ms_per_epoch_eager"] = pn
    out[f"localworld_p{n_parts}_peak_alloc_growth_gb"] = mem
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    p.add_argument("--workloads", default="rmat-1m,reddit-shaped")
    p.add_argument("--parts", default="1,4")
    p.add_argument("--leg", default=None, help=argparse.SUPPRESS)      # shape:P, run in a child process
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("genconv_bench needs a CUDA device")
    torch.cuda.set_device(0)
    if a.leg is not None:
        shape, n_parts = a.leg.split(":")
        print(json.dumps(bench_leg(shape, int(n_parts), a)))
        return
    result = dict(card=card())
    print(json.dumps(result), flush=True)
    for shape in a.workloads.split(","):
        wl = WORKLOADS[shape]
        res = dict(workload=f"{wl['n_layers']} layers, hidden 256, {wl['dtype']}, --enable-pipeline, dropout 0.5")
        for n_parts in (int(x) for x in a.parts.split(",")):
            cmd = [sys.executable, __file__, "--leg", f"{shape}:{n_parts}", "--epochs", str(a.epochs), "--rounds",
                   str(a.rounds), "--launches", str(a.launches)]
            run = subprocess.run(cmd, capture_output=True, text=True)
            if run.returncode == 0:
                leg = json.loads(run.stdout.strip().splitlines()[-1])
            else:
                tail = (run.stderr.strip().splitlines() or ["?"])[-1]
                leg = {f"p{n_parts}": f"not measured: {tail[:300]}"}
            res.update(leg)
            print(json.dumps({shape: leg}), flush=True)
        result[shape] = res
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
