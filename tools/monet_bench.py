"""Gaussian mixture model convolution (`--model monet`, K = 3) against graph convolution (`--model graphconv`) and
GraphSAGE-mean on one GPU, and the MoNet kernels alone.

    python tools/monet_bench.py [--epochs 10] [--rounds 3] [--launches 50] [--workloads rmat-1m,reddit-shaped]

Workloads (--enable-pipeline, dropout 0.5, P = 1, device-timed CUDA-graph replay): rmat-1m with 3 layers of 256 in
bf16, and reddit-shaped with 4 layers of 256 in fp32.  At K = 3 both cover both evaluation orders: layer 0 and the
hidden layers aggregate first (d_in <= 3 d_out: 256 <= 768, 602 <= 768), the logit layers transform first (256 > 3 *
64 = 192, 256 > 3 * 41 = 123).  The three models run in the same process on the same graph, alternating round by
round, so that all see the same clocks; the growth of the device's peak allocation while each model is built and run
is its memory (MoNet's aggregate-first layers keep A [N, 3 d_in] for the weight gradient).  The kernel section times
each MoNet pass on the P = 1 graph at a hidden layer's shape (d_in = d_out = 256: the aggregate-first forward and
backward gathers) and at the logit layer's (d_in = 256, d_out = n_class: the transform-first gathers), in the
workload's dtype, and states its algorithmic bytes, computed from shapes, against the H100 SXM data-sheet HBM3
bandwidth (3.35 TB/s).  The card's name, power limit and max SM clock are read in the same call.  Every workload runs
in a process of its own; each leg's JSON line is printed as it finishes, then one JSON object of all.
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
MODELS = ("monet", "graphconv", "graphsage")
K = 3


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
                              monet_kernels=K)


def timed(fn, epochs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(epochs):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / epochs


def monet_bytes(graph, d_in, d_out, es):
    """Algorithmic bytes of one launch of each MoNet pass, activation element size es, N inner rows, U all rows, E
    edges: 4 bytes of column id, and two of c and 1/deg, per edge; aggregate first (hidden shape) es d_in per edge plus
    es K d_in per row (the forward writes A [N, K d_in], the backward reads dA at the edges and h at every row and
    writes dh [U, d_in]); transform first (logit shape) es K d_out per edge (the forward gathers z's K slices, the
    backward G at the edges and z at every row, and writes dz [U, K d_out])."""
    n, u, e = graph.num_in, graph.num_all, graph.nnz
    idx = 12 * e
    return {
        "pg_monet_agg_k": idx + es * d_in * e + es * K * d_in * n,
        "pg_monet_bwd_sum": idx + es * K * d_in * e + 2 * es * d_in * u,
        "pg_monet_agg_sum": idx + es * K * d_out * e + es * d_out * n,
        "pg_monet_bwd_k": idx + es * d_out * e + 2 * es * K * d_out * u,
    }


def kernel_times(graph, dtype, d_logit, launches):
    from pipegcn_b200 import ops
    from pipegcn_b200.graph import alloc_rows
    d = 256
    n, u = graph.num_in, graph.num_all
    gen = torch.Generator(device="cuda").manual_seed(0)

    def rnd(rows, cols):
        t = alloc_rows(rows, cols, dtype, "cuda")
        t.copy_(torch.randn(rows, cols, generator=gen, device="cuda"))
        return t

    mu = (0.5 + 0.1 * torch.randn(K, 2, generator=gen, device="cuda")).contiguous()
    isg = torch.ones(K, 2, device="cuda")
    sl = ops.monet_slice(d_logit, dtype)
    h, da = rnd(u, d), rnd(n, K * d)
    z, g = rnd(u, K * sl), rnd(n, d_logit)
    calls = {
        "pg_monet_agg_k": lambda: ops.monet_agg_k(graph, h, mu, isg),
        "pg_monet_bwd_sum": lambda: ops.monet_bwd_sum(graph, da, h, mu, isg),
        "pg_monet_agg_sum": lambda: ops.monet_agg_sum(graph, z, d_logit, mu, isg),
        "pg_monet_bwd_k": lambda: ops.monet_bwd_k(graph, g, z, mu, isg),
    }
    nbytes = monet_bytes(graph, d, d_logit, h.element_size())
    res = {}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        ms = timed(fn, launches)
        shape = f"d_in {d}, d_out {d}" if name in ("pg_monet_agg_k", "pg_monet_bwd_sum") else \
            f"d_in {d}, d_out {d_logit}"
        res[name] = dict(shape=shape, ms=round(ms, 4), bytes=int(nbytes[name]), gbps=round(nbytes[name] / ms / 1e6, 1),
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
            "kernels": kernel_times(engines["monet"].graph, dtype, int(g.label.max()) + 1, a.launches)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--launches", type=int, default=50)
    p.add_argument("--workloads", default="rmat-1m,reddit-shaped")
    p.add_argument("--leg", default=None, help=argparse.SUPPRESS)      # a workload, run in a child process
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("monet_bench needs a CUDA device")
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
