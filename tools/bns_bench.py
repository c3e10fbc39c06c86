"""Boundary-node sampling (`--sampling-rate p`): halo bytes pushed per epoch and milliseconds per epoch of synchronous
training for p in {1, 0.5, 0.1}.

    python tools/bns_bench.py [--shapes rmat-1m reddit-shaped] [--rates 1 0.5 0.1] [--parts 4] [--epochs 10]
    torchrun --nproc-per-node N tools/bns_bench.py [--shapes ...]        # one partition per GPU

One GPU: a LocalWorld of --parts partitions on that GPU (the partitions run one after another on one device, and the
"NVLink" pushes are stores into the same memory, so the time saved is the copy work, not link time).  Under torchrun
every rank holds one partition on its own GPU.  Bytes are counted from the message descriptors and the keep masks of
the timed epochs: every kept halo row of every exchanged graph layer once forward and, for layers >= 1, once backward.
Prints one JSON line per (shape, p).  `--check` also asserts, every epoch, that the loss is finite and that every
unkept halo row of every exchanged layer reads as zero (prints "BNS CHECK OK").
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIG = {"rmat-1m": dict(n_layers=3, n_hidden=256), "reddit-shaped": dict(n_layers=4, n_hidden=256),
          "tiny": dict(n_layers=3, n_hidden=16), "small": dict(n_layers=3, n_hidden=64)}


def _args(g, shape, dtype, rate):
    from pipegcn_b200.synthetic import SHAPES
    base = dict(model="graphsage", backend="nccl", dtype=dtype, n_linear=0, n_feat=g.n_feat,
                n_class=SHAPES[shape]["n_class"], n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2,
                weight_decay=0.0, use_pp=False, enable_pipeline=False, feat_corr=False, grad_corr=False,
                corr_momentum=0.95, seed=0, n_epochs=1, log_every=1, **CONFIG.get(shape, CONFIG["small"]))
    if rate < 1.0:
        base["sampling_rate"] = rate
    return argparse.Namespace(**base)


def halo_bytes(buf):
    """Bytes the peers push into this rank's halo rows in the current epoch: kept rows x (forward width + backward
    width) over the exchanged graph layers (layer 0 with the static store is exchanged once, not per epoch)."""
    n_halo = buf._num_all - buf._num_in
    kept = int(buf.sample_mask().sum().item()) if buf.sampling else n_halo
    per_row = 0
    for layer, d in enumerate(buf._layer_size):
        if (layer, 0) not in buf._f_off or (layer == 0 and buf.static0_ready):
            continue
        per_row += d * buf._es * (2 if layer > 0 else 1)
    return kept * per_row, kept, n_halo


def _check(engines, losses):
    for e, loss in zip(engines, losses):
        assert torch.isfinite(loss).all(), "non-finite loss"
        buf = e.buffer
        if not buf.sampling:
            continue
        dead = ~buf.sample_mask()
        for (layer, v), rows in buf._f_buf.items():
            halo = rows[buf._num_in:, :buf._layer_size[layer]]
            assert not halo[dead].any(), f"rank {buf._world.rank} layer {layer}: an unkept halo row is not zero"


def run_local(g, layouts, shape, rate, args_ns):
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    P = len(layouts)
    args = _args(g, shape, args_ns.dtype, rate)
    tr = LocalTrainer(layouts, args, LocalWorld(P, "cuda"))
    for _ in range(args_ns.warmup):
        tr.run_epoch()
    torch.cuda.synchronize()
    ms, nbytes, kept, halo = [], 0, 0, 0
    for _ in range(args_ns.epochs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        losses = tr.run_epoch()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        if args_ns.check:
            _check(tr.engines, losses)
        for e in tr.engines:
            b, k, h = halo_bytes(e.buffer)
            nbytes, kept, halo = nbytes + b, kept + k, halo + h
    for e in tr.engines:
        e.buffer.release()
    return ms, nbytes, kept, halo


def run_dist(g, layouts, shape, rate, args_ns, world):
    import torch.distributed as dist
    from pipegcn_b200.train import RankEngine
    args = _args(g, shape, args_ns.dtype, rate)
    eng = RankEngine(layouts[world.rank], args, world)
    for _ in range(args_ns.warmup):
        eng.run_epoch()
    torch.cuda.synchronize()
    dist.barrier()
    ms, nbytes, kept, halo = [], 0, 0, 0
    for _ in range(args_ns.epochs):
        t0 = time.perf_counter()
        loss = eng.run_epoch()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
        eng.buffer.check_status()
        if args_ns.check:
            _check([eng], [loss])
        b, k, h = halo_bytes(eng.buffer)
        nbytes, kept, halo = nbytes + b, kept + k, halo + h
    tot = torch.tensor([nbytes, kept, halo], dtype=torch.float64, device=world.device)
    dist.all_reduce(tot)
    worst = torch.tensor([sorted(ms)[len(ms) // 2]], device=world.device)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    eng.buffer.synchronize()
    torch.cuda.synchronize()
    eng.buffer.release()
    return [float(worst.item())], int(tot[0].item()), int(tot[1].item()), int(tot[2].item())


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", nargs="+", default=["rmat-1m", "reddit-shaped"])
    ap.add_argument("--rates", nargs="+", type=float, default=[1.0, 0.5, 0.1])
    ap.add_argument("--parts", type=int, default=4, help="partitions of the one-GPU LocalWorld")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dtype", choices=["fp32", "bf16"], default="fp32")
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
    gpu = torch.cuda.get_device_name(0)
    for shape in a.shapes:
        g = make_graph(shape)
        layouts = build_layouts(g, random_partition(g.n_nodes, P), P)
        base = None
        for rate in a.rates:
            if dist_run:
                ms, nbytes, kept, halo = run_dist(g, layouts, shape, rate, a, world)
            else:
                ms, nbytes, kept, halo = run_local(g, layouts, shape, rate, a)
            ms.sort()
            per_epoch = nbytes / a.epochs
            if base is None and rate == 1.0:
                base = per_epoch
            if rank0:
                print(json.dumps({
                    "shape": shape, "P": P, "mode": "torchrun" if dist_run else "LocalWorld, one GPU",
                    "sampling_rate": rate, "dtype": a.dtype, "ms_per_epoch_median": round(ms[len(ms) // 2], 3),
                    "halo_bytes_pushed_per_epoch": int(per_epoch),
                    "bytes_vs_p1": round(per_epoch / base, 4) if base else None,
                    "kept_halo_rows_fraction": round(kept / max(halo, 1), 4), "epochs": a.epochs, "gpu": gpu}),
                    flush=True)
        del g, layouts
        torch.cuda.empty_cache()
    if a.check and rank0:
        print("BNS CHECK OK", flush=True)
    if dist_run:
        import torch.distributed as dist
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
