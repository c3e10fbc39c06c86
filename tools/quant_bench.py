"""Quantised halo messages (`--halo-bits`): link bytes, epoch time, kernel time and accuracy against exact messages.

    python tools/quant_bench.py [--shapes rmat-1m reddit-shaped] [--bits 0 8 4] [--parts 4] [--epochs 10]
    torchrun --nproc-per-node N tools/quant_bench.py [--shapes ...]        # one partition per GPU

For every (shape, dtype, exchange mode, bits) it prints one JSON line with
1. the link bytes pushed per epoch, counted from the messages every rank pushes (halo rows x (code row + 8 bytes) for
   the quantised layers >= 1, rows x d x element size for the exact ones; layer 0 with the static store is exchanged
   once, not per epoch);
2. the median ms per epoch over --epochs eager epochs after --warmup;
3. per launch (CUDA events over 50 launches, on rank 0's layer-1 messages): pg_halo_push_q + pg_halo_dequant against
   pg_halo_push, and pg_boundary_add_q against pg_boundary_add.
Then, on `small` with planted labels, the train loss and validation accuracy after --acc-epochs epochs for each bits.
The card's name and power limit are read in the same run and printed.

One GPU: a LocalWorld of --parts partitions on that GPU.  Its "link" is a store into the same card's memory, so the
bytes shrink by the code ratio while the time saved is copy work only, and the decode adds a pass: expect the time to
be about even or slightly slower.  A multi-GPU speed-up needs torchrun on several GPUs.  `--check` asserts that every
loss is finite (prints "QUANT CHECK OK").
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIG = {"rmat-1m": dict(n_layers=3, n_hidden=256), "reddit-shaped": dict(n_layers=4, n_hidden=256),
          "tiny": dict(n_layers=3, n_hidden=16), "small": dict(n_layers=3, n_hidden=64)}
MODES = {"sync": dict(), "pipeline": dict(enable_pipeline=True)}


def _args(g, shape, dtype, bits, mode, **kw):
    from pipegcn_b200.synthetic import SHAPES
    base = dict(model="graphsage", backend="nccl", dtype=dtype, n_linear=0, n_feat=g.n_feat,
                n_class=SHAPES[shape]["n_class"], n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2,
                weight_decay=0.0, use_pp=False, enable_pipeline=False, feat_corr=False, grad_corr=False,
                corr_momentum=0.95, seed=0, n_epochs=1, log_every=1, **CONFIG.get(shape, CONFIG["small"]))
    base.update(MODES[mode])
    base.update(kw)
    if bits:
        base["halo_bits"] = bits
    return argparse.Namespace(**base)


def link_bytes(buf):
    """Bytes this rank pushes in one epoch: its boundary rows forward and its halo rows' gradients backward, per
    exchanged graph layer."""
    from pipegcn_b200.ops import quant_link_bytes
    fwd = sum(int(buf._bidx[j].numel()) for j in buf._peers)
    bwd = sum(int(buf._recv_shape[j]) for j in buf._peers)
    total = 0
    for layer, d in enumerate(buf._layer_size):
        if (layer, 0) not in buf._f_off or (layer == 0 and buf.static0_ready):
            continue
        bits = buf.halo_bits if layer > 0 else None
        total += quant_link_bytes(fwd, d, bits, buf._es)
        if layer > 0:
            total += quant_link_bytes(bwd, d, bits, buf._es)
    return total


def _events(fn, n=50):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def kernel_us(buf, bits, dtype):
    """Per-launch microseconds of the exact and quantised kernels on this rank's layer-1 message shapes (local
    destinations)."""
    from pipegcn_b200 import _C, ops
    from pipegcn_b200.helper.feature_buffer import _MsgSet
    d = buf._layer_size[1]
    ld = (d + 7) // 8 * 8
    dev = buf._world.device
    idx = torch.cat([buf._bidx[j] for j in buf._peers])
    n = int(idx.numel())
    src = torch.randn(buf._num_in, ld, device=dev).to(dtype)
    dst = torch.zeros(n, ld, device=dev, dtype=dtype)
    qld = ops.quant_row_bytes(d, bits)
    codes = torch.zeros(n, qld, dtype=torch.uint8, device=dev)
    pairs = torch.zeros(n, 2, device=dev)
    ms = _MsgSet([_C.pg_msg(idx.data_ptr(), 0, n, 0, dst.data_ptr(), ld, None, 0, None, None, 0)], dev)
    mq = _MsgSet([_C.pg_msg(idx.data_ptr(), 0, n, 0, codes.data_ptr(), qld, None, 0, None, None, 0)], dev)
    qm = ops.qmsg_array([(pairs.data_ptr(), 1)], dev)
    spec = ops.QuantSpec(bits, 1, 1, 0)
    code = _C.dtype_code(dtype)
    out = torch.zeros(n, ld, device=dev, dtype=dtype)
    push = _events(lambda: _C.lib.pg_halo_push(ms.ptr, 1, ms.n_ctas, src.data_ptr(), ld, d, code, 0.0, 1.0, 1, None,
                                               _C.stream_ptr()))
    push_q = _events(lambda: ops.halo_push_q(mq, qm, src, d, spec, 1))
    deq = _events(lambda: ops.halo_dequant(codes, pairs, d, bits, out))
    res = dict(push_us=round(push, 2), push_q_us=round(push_q, 2), dequant_us=round(deq, 2),
               push_q_plus_dequant_us=round(push_q + deq, 2))
    if buf._urow is not None:
        btot = int(buf._usrc.numel())
        grad = torch.randn(buf._num_all, ld, device=dev).to(dtype)
        recv = torch.randn(btot, ld, device=dev).to(dtype)
        bcodes = torch.randint(0, 255, (btot, qld), dtype=torch.uint8, device=dev)
        bpairs = torch.rand(btot, 2, device=dev)
        args = (buf._urow.data_ptr(), buf._uptr.data_ptr(), buf._usrc.data_ptr(), int(buf._urow.numel()))
        res["boundary_add_us"] = round(_events(lambda: _C.lib.pg_boundary_add(
            grad.data_ptr(), ld, recv.data_ptr(), ld, d, code, *args, _C.stream_ptr())), 2)
        res["boundary_add_q_us"] = round(_events(lambda: ops.boundary_add_q(
            grad, d, bcodes, bpairs, bits, buf._urow, buf._uptr, buf._usrc)), 2)
    return res


def run_local(g, layouts, args, a):
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    tr = LocalTrainer(layouts, args, LocalWorld(len(layouts), "cuda"))
    for _ in range(a.warmup):
        tr.run_epoch()
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.epochs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        losses = tr.run_epoch()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        if a.check:
            assert all(torch.isfinite(x).all() for x in losses), "non-finite loss"
    nbytes = sum(link_bytes(e.buffer) for e in tr.engines)
    kern = None
    if getattr(args, "halo_bits", None) and len(layouts) > 1:
        kern = kernel_us(tr.engines[0].buffer, args.halo_bits, tr.engines[0].dtype)
    for e in tr.engines:
        e.buffer.release()
    return ms, nbytes, kern


def run_dist(g, layouts, args, a, world):
    import torch.distributed as dist
    from pipegcn_b200.train import RankEngine
    eng = RankEngine(layouts[world.rank], args, world)
    for _ in range(a.warmup):
        eng.run_epoch()
    torch.cuda.synchronize()
    dist.barrier()
    ms = []
    for _ in range(a.epochs):
        t0 = time.perf_counter()
        loss = eng.run_epoch()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
        eng.buffer.check_status()
        if a.check:
            assert torch.isfinite(loss).all(), "non-finite loss"
    tot = torch.tensor([link_bytes(eng.buffer)], dtype=torch.float64, device=world.device)
    dist.all_reduce(tot)
    worst = torch.tensor([sorted(ms)[len(ms) // 2]], device=world.device)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    eng.buffer.synchronize()
    torch.cuda.synchronize()
    eng.buffer.release()
    return [float(worst.item())], int(tot[0].item()), None


def accuracy(bits, a, P):
    """Train loss (summed over ranks, / n_train) and validation accuracy after a.acc_epochs pipelined epochs on the
    planted labels of `small`."""
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    g = make_graph("small", planted_labels=True)
    layouts = build_layouts(g, random_partition(g.n_nodes, P), P)
    args = _args(g, "small", "fp32", bits, "pipeline", dropout=0.2)
    tr = LocalTrainer(layouts, args, LocalWorld(P, "cuda"))
    for _ in range(a.acc_epochs):
        losses = tr.run_epoch()
    loss = sum(float(x) for x in losses) / args.n_train
    hit = tot = 0
    for z, lay in zip(tr.predict(), layouts):
        m = lay.val_mask.to("cuda")
        hit += int((z.float().argmax(1)[m] == lay.label.to("cuda")[m]).sum())
        tot += int(m.sum())
    tr.release_eval()
    for e in tr.engines:
        e.buffer.release()
    return loss, hit / tot


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:                        # the name from torch is still reported
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", nargs="+", default=["rmat-1m", "reddit-shaped"])
    ap.add_argument("--bits", nargs="+", type=int, default=[0, 8, 4], help="0 = exact messages")
    ap.add_argument("--dtypes", nargs="+", default=["fp32", "bf16"])
    ap.add_argument("--modes", nargs="+", default=list(MODES))
    ap.add_argument("--parts", type=int, default=4, help="partitions of the one-GPU LocalWorld")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--acc-epochs", type=int, default=60, help="0: skip the accuracy runs")
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    dist_run = "RANK" in os.environ
    world = None
    if dist_run:
        import torch.distributed as dist
        from pipegcn_b200.world import DistWorld
        local = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dev = torch.device(f"cuda:{local}")
        dist.init_process_group("nccl", rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]),
                                device_id=dev)
        world = DistWorld(device=dev)
    P = world.size if dist_run else a.parts
    rank0 = not dist_run or world.rank == 0
    gpu = card()
    if rank0:
        print(json.dumps({"gpu": gpu}), flush=True)
    for shape in a.shapes:
        g = make_graph(shape)
        layouts = build_layouts(g, random_partition(g.n_nodes, P), P)
        for dtype in a.dtypes:
            for mode in a.modes:
                base = None
                for bits in a.bits:
                    args = _args(g, shape, dtype, bits, mode)
                    if dist_run:
                        ms, nbytes, kern = run_dist(g, layouts, args, a, world)
                    else:
                        ms, nbytes, kern = run_local(g, layouts, args, a)
                    gc.collect()                  # the trainer's reference cycles hold device memory
                    torch.cuda.empty_cache()
                    ms.sort()
                    med = ms[len(ms) // 2]
                    if base is None:
                        base = (nbytes, med)
                    if rank0:
                        print(json.dumps({
                            "shape": shape, "P": P, "mode": mode, "world": "torchrun" if dist_run else "LocalWorld, one GPU",
                            "dtype": dtype, "halo_bits": bits or "exact", "link_bytes_per_epoch": nbytes,
                            "bytes_vs_first": round(nbytes / base[0], 4) if base[0] else None,
                            "ms_per_epoch_median": round(med, 3), "ms_vs_first": round(med / base[1], 4),
                            "kernels": kern, "epochs": a.epochs, "gpu": gpu}), flush=True)
        del g, layouts
        torch.cuda.empty_cache()
    if a.acc_epochs and not dist_run:
        for bits in a.bits:
            loss, acc = accuracy(bits, a, P)
            print(json.dumps({"accuracy": "small, planted labels", "P": P, "dtype": "fp32", "halo_bits": bits or "exact", "epochs": a.acc_epochs,
                              "train_loss": round(loss, 4), "val_acc": round(acc, 4), "gpu": gpu}), flush=True)
    if a.check and rank0:
        print("QUANT CHECK OK", flush=True)
    if dist_run:
        import torch.distributed as dist
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
