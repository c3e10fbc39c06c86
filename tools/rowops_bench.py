"""Time the row kernels alone (LayerNorm+ReLU(+dropout) forward, its backward, stand-alone dropout) on one GPU.

    python tools/rowops_bench.py [--rows 1048576] [--d 256] [--dtype bf16] [--iters 20]

Prints one JSON line per (kernel, ln_stage): milliseconds per launch (CUDA events, L2 flushed between launches by
the working set itself: every tensor is larger than the 50 MB L2 at the default size) and the HBM GB/s of the
algorithmic bytes (tensors read once + written once).
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
    ap.add_argument("--d", type=int, default=256)
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--p", type=float, default=0.5)
    a = ap.parse_args()
    from pipegcn_b200 import _C, ops
    from pipegcn_b200.graph import alloc_rows
    dt = torch.bfloat16 if a.dtype == "bf16" else torch.float32
    dev = "cuda"
    n, d, es = a.rows, a.d, (2 if a.dtype == "bf16" else 4)
    torch.manual_seed(0)
    y = alloc_rows(n, d, dt, dev)
    y.copy_(torch.randn(n, d, device=dev))
    g = alloc_rows(n, d, dt, dev)
    g.copy_(torch.randn(n, d, device=dev))
    gamma, beta = torch.rand(d, device=dev) + 0.5, torch.randn(d, device=dev)
    out, clean = alloc_rows(n, d, dt, dev), alloc_rows(n, d, dt, dev)
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    spec = ops.DropSpec(a.p, 4242, step, 0)
    tensor_bytes = n * d * es

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(a.iters + 1)]
        ev[0].record()
        for i in range(a.iters):
            fn()
            ev[i + 1].record()
        torch.cuda.synchronize()
        ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(a.iters))
        return ts[len(ts) // 2], ts[0]

    for stage in (1, 0):
        _C.check(_C.lib.pg_set_option(b"ln_stage", stage))
        cases = {
            "ln_relu_fwd": (lambda: ops.layer_norm_relu(y, gamma, beta, 1e-5, True, out), 2),
            "ln_relu_drop_fwd": (lambda: ops.layer_norm_relu(y, gamma, beta, 1e-5, True, out, None, spec), 2),
            "ln_relu_drop_clean_fwd": (lambda: ops.layer_norm_relu(y, gamma, beta, 1e-5, True, out, clean, spec), 3),
        }
        yq = y.detach().requires_grad_(True)
        gq, bq = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        o = ops.layer_norm_relu(yq, gq, bq, 1e-5, True, out)

        def bwd():
            yq.grad = None
            o.backward(g, retain_graph=True)
        cases["ln_relu_bwd"] = (bwd, 3)
        for name, (fn, n_tensors) in cases.items():
            med, best = timed(fn)
            print(json.dumps(dict(kernel=name, ln_stage=stage, rows=n, d=d, dtype=a.dtype, ms=round(med, 4),
                                  ms_best=round(best, 4), gbs=round(n_tensors * tensor_bytes / med / 1e6, 1))), flush=True)
    _C.lib.pg_set_option(b"ln_stage", 1)
    med, best = timed(lambda: ops.dropout_rows(y, spec))
    print(json.dumps(dict(kernel="dropout_rows", rows=n, d=d, dtype=a.dtype, ms=round(med, 4), ms_best=round(best, 4),
                          gbs=round(2 * tensor_bytes / med / 1e6, 1))), flush=True)


if __name__ == "__main__":
    main()
