"""Aggregate kernel benchmark on one partition of a P-way split of a named shape (what a rank of a P-GPU run executes):
forward (CSR by destination, with the division) and backward (CSC by source, accumulate) for the kernel variants
(`agg_impl` 1 = row per lane group; 2 = chunked; 3 = chunked with the long rows staged through shared memory by
cp.async; n/h = without/with L2 eviction hints; 4/5 = CTAs per SM the register-landing long-row kernel is built for;
trailing s = short-row kernel serialised after the long-row kernel instead of on a side stream, trailing w = rows of
at most 16 vectors through the row-per-group kernel instead of the chunked sub-warp kernels),
CUDA-event timed, checked against cuSPARSE (fp32 SpMM); one JSON line per variant.

    python tools/agg_bench.py [shape=rmat-1m] [P=1] [dtype=bf16] [d=n_feat] [--once] [--variants 1,2h4,...]
`--once`: a single launch per case after warm-up (for a profiler run).
"""
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch

from bench import peaks
from pipegcn_b200 import _C, ops
from pipegcn_b200.graph import PartGraph, alloc_rows
from pipegcn_b200.partition import PartitionPlan
from pipegcn_b200.synthetic import make_graph, random_partition

HBM_PEAK, PEAK_SOURCE = peaks()      # the denominator bench.py uses
argv = [a for a in sys.argv[1:] if not a.startswith("--")]
once = "--once" in sys.argv
variants = ["1", "2n4s", "2h4s", "2n4", "2h4"]
if "--variants" in sys.argv:
    variants = sys.argv[sys.argv.index("--variants") + 1].split(",")
    argv = [a for a in argv if a != ",".join(variants)]
shape = argv[0] if len(argv) > 0 else "rmat-1m"
P = int(argv[1]) if len(argv) > 1 else 1
dtype = {"bf16": torch.bfloat16, "fp32": torch.float32}[argv[2] if len(argv) > 2 else "bf16"]
g = make_graph(shape, device="cuda")
d = int(argv[3]) if len(argv) > 3 else g.n_feat
part = random_partition(g.n_nodes, P, seed=1, device="cuda")
lay = PartitionPlan(g, part, P).build(0)
del g
graph = PartGraph.from_layout(lay, device="cuda")
x = alloc_rows(lay.num_all, d, dtype, "cuda")
x.copy_(torch.randn(lay.num_all, d, device="cuda"))
gy = alloc_rows(lay.num_in, d, dtype, "cuda")
gy.copy_(torch.randn(lay.num_in, d, device="cuda"))
gx = alloc_rows(lay.num_all, d, dtype, "cuda", zero=True)
info = dict(shape=shape, P=P, dtype=str(dtype), d=d, n_in=lay.num_in, num_all=lay.num_all, nnz=lay.nnz,
            chunks_fwd=graph.fwd.n_chunks, chunks_long_fwd=graph.fwd.n_chunks_long, hot_fwd=graph.fwd.n_hot,
            chunks_bwd=graph.bwd.n_chunks, seg_len=graph.fwd.seg_len)


def spmm_ref(plan, xin, n_cols):
    a = torch.sparse_csr_tensor(plan.indptr.to(torch.int64), plan.indices.to(torch.int64),
                                torch.ones(plan.nnz, device="cuda"), size=(plan.n_rows, n_cols))
    return a @ xin.float()


ref_f = spmm_ref(graph.fwd, x, lay.num_all) / graph.in_deg_f[:, None]
ref_b = spmm_ref(graph.bwd, gy, lay.num_in)
tol = 2e-5 if dtype == torch.float32 else 1.6e-2


def timeit(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    if once:
        n = 1
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for var in variants:
    impl = int(var[0])
    _C.check(_C.lib.pg_set_option(b"agg_impl", impl))
    if impl >= 2:
        _C.check(_C.lib.pg_set_option(b"agg_l2_hint", 1 if var[1] == "h" else 0))
        _C.check(_C.lib.pg_set_option(b"agg_occ", int(var[2])))
        _C.check(_C.lib.pg_set_option(b"agg_overlap", 0 if "s" in var[3:] else 1))
        _C.check(_C.lib.pg_set_option(b"agg_narrow", 0 if "w" in var[3:] else 1))
    of = ops.aggregate(graph.fwd, x, row_div=graph.in_deg_f)
    ob = ops.aggregate(graph.bwd, gy, out=torch.zeros_like(gx), acc_rows=0)
    err_f = ((of.float() - ref_f).abs().max() / ref_f.abs().max()).item()
    err_b = ((ob.float() - ref_b).abs().max() / ref_b.abs().max()).item()
    tf = timeit(lambda: ops.aggregate(graph.fwd, x, row_div=graph.in_deg_f))
    tb = timeit(lambda: ops.aggregate(graph.bwd, gy, out=gx, acc_rows=lay.num_in))
    bf = ops.aggregate_bytes(graph.fwd, x, True)
    bb = ops.aggregate_bytes(graph.bwd, gy, False)
    es = x.element_size()
    print(json.dumps(dict(info, variant=var, ok=bool(err_f <= tol and err_b <= tol), err_fwd=err_f, err_bwd=err_b,
                          fwd_ms=tf, bwd_ms=tb, fwd_frac_of_hbm_peak=bf / tf / 1e6 / HBM_PEAK, bwd_frac_of_hbm_peak=bb / tb / 1e6 / HBM_PEAK,
                          hbm_peak_gbs=HBM_PEAK, hbm_peak_source=PEAK_SOURCE,
                          fwd_gather_tbs=lay.nnz * d * es / tf / 1e9, bwd_gather_tbs=lay.nnz * d * es / tb / 1e9)), flush=True)
_C.lib.pg_set_option(b"agg_impl", 2)
_C.lib.pg_set_option(b"agg_l2_hint", 0)
_C.lib.pg_set_option(b"agg_occ", 4)
_C.lib.pg_set_option(b"agg_overlap", 1)
_C.lib.pg_set_option(b"agg_narrow", 1)
