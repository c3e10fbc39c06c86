"""Time pg_linear alone on the shapes of the headline workload, with one and two epilogue staging slabs per warp.

    python tools/gemm_bench.py [--rows 1048576] [--dtype bf16] [--iters 20]

One JSON line per (K, N, gemm_epi_slabs): median ms per launch (CUDA events) and GB/s of operand + result bytes.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    from pipegcn_b200 import _C, ops
    from pipegcn_b200.graph import alloc_rows
    dt = torch.bfloat16 if a.dtype == "bf16" else torch.float32
    es = 2 if a.dtype == "bf16" else 4
    m = a.rows
    torch.manual_seed(0)
    for k_list, n in (([256, 256], 256), ([256], 256), ([64, 64], 256), ([256], 128), ([256], 64)):
        xs = []
        for k in k_list:
            x = alloc_rows(m, k, dt, "cuda")
            x.copy_(torch.randn(m, k, device="cuda"))
            xs.append(x)
        ws = [ops.padded_weight(torch.randn(n, k, device="cuda") * 0.05, dt) for k in k_list]
        out = alloc_rows(m, n, dt, "cuda")
        args = [xs[0], ws[0]] + ([xs[1], ws[1]] if len(xs) > 1 else [])
        for slabs in (2, 1, 2, 1):
            _C.check(_C.lib.pg_set_option(b"gemm_epi_slabs", slabs))
            for _ in range(3):
                ops.gemm_nt(*args, out=out)
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(a.iters + 1)]
            ev[0].record()
            for i in range(a.iters):
                ops.gemm_nt(*args, out=out)
                ev[i + 1].record()
            torch.cuda.synchronize()
            ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(a.iters))
            med = ts[len(ts) // 2]
            nbytes = m * (sum(k_list) + n) * es
            print(json.dumps(dict(kernel="linear_wgmma", k=k_list, n=n, rows=m, dtype=a.dtype, gemm_epi_slabs=slabs,
                                  ms=round(med, 4), ms_best=round(ts[0], 4), gbs=round(nbytes / med / 1e6, 1))), flush=True)
    _C.lib.pg_set_option(b"gemm_epi_slabs", 2)


if __name__ == "__main__":
    main()
