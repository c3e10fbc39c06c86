"""Per-kernel time and HBM traffic of one bench.py epoch.

    python tools/step_profile.py [--workload rmat-1m] [--warmup 5] [--epochs 3] [--out DIR]

Builds the workload exactly as `bench.py --gpus 1` does (same engine arguments, graph, seeds and partition), runs
warm-up epochs, then profiles a few eager (Python-launched) epochs with torch.profiler (CUDA activities).  Writes
DIR/kernels.json and DIR/kernels.md: per kernel the calls and total time, and per kernel family (GEMM, weight gradient,
aggregate, row kernels) the algorithmic bytes per epoch -- computed from the shapes the library was called with -- and
the achieved GB/s.  The card's name and power limit are read in the same run and written beside the numbers.
`--dry-run` builds a scaled-down graph on the host and prints its layout's shapes without a device (argument and
shape checking only: no time is measured).
"""
from __future__ import annotations

import argparse
import json
import re
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

# kernel family: (kernel-name pattern, library calls whose bytes it carries)
FAMILIES = [
    ("gemm", r"linear_wgmma", ("pg_linear", "pg_linear_drop", "pg_linear_group")),
    ("wgrad", r"wgrad_", ("pg_wgrad", "pg_wgrad_group")),
    ("aggregate", r"agg", ("aggregate",)),
    ("ln_relu", r"ln_relu", ("pg_ln_relu_fwd", "pg_ln_relu_drop_fwd", "pg_ln_relu_bwd", "pg_ln_relu_bwd2")),
    ("cross_entropy", r"ce_(fwd|bwd)", ("pg_ce_fwd", "pg_ce_bwd")),
    ("dropout", r"dropout_kernel", ("pg_dropout", "pg_dropout_rows")),
    ("row_div", r"row_div", ("pg_row_div",)),
    ("split_tf32", r"split_tf32", ("pg_split_tf32",)),
]
ES = {0: 4, 1: 2}     # PG_F32, PG_BF16


def _unique_rows(ptrs_and_bytes):
    seen, total = set(), 0
    for ptr, nb in ptrs_and_bytes:
        if ptr not in seen:
            seen.add(ptr)
            total += nb
    return total


def _linear_bytes(es_in, es_out, srcs, n_src, m, n, rows_div, outs):
    """A once per distinct operand, every B once, every output written once (+ the row divisors)."""
    a = _unique_rows((srcs[s].a, m * srcs[s].k * es_in) for s in range(n_src))
    b = _unique_rows((srcs[s].b, n * srcs[s].k * es_in) for s in range(len(srcs)))
    return a + b + outs * m * n * es_out + rows_div * 4 * m


def _wgrad_bytes(srcs, n_src, probs):
    """Both operands of every problem once (distinct arrays), the split-K partials written and read back, the
    fp32 output written.  `probs`: (m, n, k, workspace floats) per problem."""
    total, pairs = 0, []
    for p, (m, n, k, ws) in enumerate(probs):
        for s in range(n_src):
            src = srcs[p * n_src + s]
            pairs += [(src.a, m * n * 2), (src.b, m * k * 2)]
        total += 2 * ws * 4 + n * k * 4
    return total + _unique_rows(pairs)


def byte_model(lib, record):
    """Wrap the library's entry points so that every call adds its algorithmic bytes to record[name]."""
    def wrap(name, nbytes):
        fn = getattr(lib, name, None)
        if fn is None:
            return

        def call(*a):
            record[name] += nbytes(*a)
            return fn(*a)
        setattr(lib, name, call)

    wrap("pg_linear", lambda di, do, srcs, ns, bias, rd, c, ldc, m, n, st:
         _linear_bytes(ES[di], ES[do], srcs, ns, m, n, rd is not None, 1))
    wrap("pg_linear_drop", lambda di, do, srcs, ns, bias, rd, c, ldc, m, n, drop, r0, st:
         _linear_bytes(ES[di], ES[do], srcs, ns, m, n, rd is not None, 1))
    wrap("pg_linear_group", lambda di, do, srcs, ns, npb, outs, m, n, st:
         _linear_bytes(ES[di], ES[do], srcs, ns, m, n, sum(outs[i].row_div is not None for i in range(npb)), npb))
    wrap("pg_wgrad", lambda di, srcs, ns, out, ldo, m, n, k, ws, wsf, st: _wgrad_bytes(srcs, ns, [(m, n, k, wsf)]))
    wrap("pg_wgrad_group", lambda di, srcs, ns, npb, outs, n, k, st:
         _wgrad_bytes(srcs, ns, [(outs[i].m, n, k, outs[i].workspace_floats) for i in range(npb)]))
    wrap("pg_ln_relu_fwd", lambda *a: (2 * ES[a[12]] * a[11] + 8) * a[10])
    wrap("pg_ln_relu_drop_fwd", lambda *a: (3 * ES[a[14]] * a[13] + 8) * a[12])
    wrap("pg_ln_relu_bwd", lambda *a: (4 * ES[a[18]] * a[17] + 8) * a[16])
    wrap("pg_ln_relu_bwd2", lambda *a: ((3 + (a[2] is not None)) * ES[a[19]] * a[18] + 8) * a[17])
    wrap("pg_ce_fwd", lambda z, ld, lab, nr, c, dt, *r: nr * (c * ES[dt] + 12))
    wrap("pg_ce_bwd", lambda z, ld, lab, lse, up, nr, nt, c, dt, *r: nr * (c * ES[dt] + 12) + nt * c * ES[dt])
    wrap("pg_dropout", lambda x, lx, o, lo, nr, d, dt, *r: 2 * nr * d * ES[dt])
    wrap("pg_dropout_rows", lambda x, lx, o, lo, r0, nr, d, dt, *r: 2 * nr * d * ES[dt])
    wrap("pg_row_div", lambda x, lx, o, lo, nr, d, dt, *r: (2 * d * ES[dt] + 4) * nr)
    wrap("pg_split_tf32", lambda x, lx, hi, lo, ld, nr, d, st: 12 * nr * d)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        return out or "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({type(e).__name__})"


def build_engine(workload, scale_down, device, dropout=0.5):
    """What bench.py main() builds for --gpus 1 (random partition with seed 1, graph generated on `device`)."""
    import bench
    from pipegcn_b200.partition import PartitionPlan
    from pipegcn_b200.synthetic import make_graph, random_partition
    w = bench.WORKLOADS[workload]
    spec = bench.shape_spec(w, scale_down * w.get("scale_down", 1))
    g = make_graph(spec, device=device)
    part = random_partition(g.n_nodes, 1, seed=1, device=device)
    layout = PartitionPlan(g, part, 1).build(0)
    eargs = bench.engine_args(w, g.n_feat, spec["n_class"], int(g.train_mask.sum().item()), 1, dropout)
    return layout, eargs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="rmat-1m")
    ap.add_argument("--scale-down", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--out", default="results/step_profile")
    ap.add_argument("--dry-run", action="store_true", help="host only: build the graph and layout, print the shapes")
    args = ap.parse_args()

    import torch
    if args.dry_run:
        layout, eargs = build_engine(args.workload, max(args.scale_down, 64), "cpu")
        print(json.dumps({"workload": args.workload, "n_in": layout.num_in, "num_all": layout.num_all,
                          "nnz": layout.nnz, "n_layers": eargs.n_layers, "n_hidden": eargs.n_hidden,
                          "dtype": eargs.dtype, "g_bytes_per_layer": layout.num_in * eargs.n_hidden *
                          (2 if eargs.dtype == "bf16" else 4)}))
        return
    assert torch.cuda.is_available(), "step_profile.py measures on a GPU"
    torch.cuda.set_device(0)
    from pipegcn_b200 import _C, ops
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import LocalWorld
    layout, eargs = build_engine(args.workload, args.scale_down, torch.device("cuda:0"))
    eargs.cuda_graph = False
    engine = RankEngine(layout, eargs, LocalWorld(1, torch.device("cuda:0")).view(0))
    del layout
    for _ in range(args.warmup):
        engine.run_epoch()
    torch.cuda.synchronize()

    record = defaultdict(int)
    byte_model(_C.lib, record)
    ops.PROFILE = []
    _C.LAUNCHES = 0
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.epochs):
            engine.run_epoch()
        torch.cuda.synchronize()
    launches = _C.LAUNCHES / args.epochs
    record["aggregate"] = sum(nb for _, _, nb in ops.PROFILE)
    ops.PROFILE = None

    kernels = defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels[ev.name]
            k[0] += 1
            k[1] += ev.device_time_total / 1e3      # us -> ms
    ep = args.epochs
    rows = sorted(({"kernel": name, "calls_per_epoch": c / ep, "ms_per_epoch": t / ep} for name, (c, t) in kernels.items()),
                  key=lambda r: -r["ms_per_epoch"])
    total_ms = sum(r["ms_per_epoch"] for r in rows)
    fams = []
    for fam, pat, calls in FAMILIES:
        members = [r for r in rows if re.search(pat, r["kernel"])]
        ms = sum(r["ms_per_epoch"] for r in members)
        nbytes = sum(record[c] for c in calls) / ep
        fams.append({"family": fam, "kernels": len(members), "launches_per_epoch": sum(r["calls_per_epoch"] for r in members),
                     "ms_per_epoch": ms, "gb_per_epoch": nbytes / 1e9,
                     "achieved_gbs": nbytes / 1e9 / (ms / 1e3) if ms > 0 else None,
                     "hbm_bound_ms_at_3350gbs": nbytes / 3.35e12 * 1e3})
    other = total_ms - sum(f["ms_per_epoch"] for f in fams)
    res = {"workload": args.workload, "card": card(), "epochs": ep, "kernel_ms_per_epoch": total_ms,
           "launches_per_epoch": launches, "families": fams, "other_ms_per_epoch": other, "kernels": rows}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "kernels.json").write_text(json.dumps(res, indent=1))
    lines = [f"card: {res['card']}; {args.workload}, {ep} eager epochs after {args.warmup} warm-up; kernel time "
             f"{total_ms:.3f} ms per epoch, {launches:.0f} launches through the library", "",
             "| family | launches | ms/epoch | GB/epoch (algorithmic) | GB/s | ms at 3.35 TB/s |", "|---|---|---|---|---|---|"]
    for f in fams:
        gbs = f"{f['achieved_gbs']:.0f}" if f["achieved_gbs"] else "-"
        lines.append(f"| {f['family']} | {f['launches_per_epoch']:.0f} | {f['ms_per_epoch']:.3f} | {f['gb_per_epoch']:.2f} | "
                     f"{gbs} | {f['hbm_bound_ms_at_3350gbs']:.3f} |")
    lines.append(f"| other (torch: Adam, copies, fills, ...) | | {other:.3f} | | | |")
    lines += ["", "| kernel | calls/epoch | ms/epoch |", "|---|---|---|"]
    lines += [f"| `{r['kernel'][:110]}` | {r['calls_per_epoch']:.0f} | {r['ms_per_epoch']:.3f} |" for r in rows[:40]]
    (out / "kernels.md").write_text("\n".join(lines) + "\n")
    print("\n".join(lines[:len(fams) + 5]))


if __name__ == "__main__":
    main()
