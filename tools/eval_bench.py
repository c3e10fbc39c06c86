"""Time the evaluation of one `log_every` step: rank 0's full-graph evaluation (`--eval`) against the
partition-parallel one (`--eval --eval-partitioned`).

    python tools/eval_bench.py [--shapes rmat-1m reddit-shaped] [--parts 1 4] [--repeat 5] [--dtype bf16]
    torchrun --nproc-per-node N tools/eval_bench.py [--shapes ...]        # the real N-GPU split

One GPU: LocalWorld P = 1 and P = 4 on that GPU (the partitions run one after another on one device, so both paths do
the same total work: expect parity, not a speed-up).  Under torchrun each rank holds one partition on its own GPU;
rank 0 also times its full-graph evaluation, which is what `--eval` runs while the other ranks wait.
Prints one JSON line per (shape, path, P): milliseconds per evaluation (CUDA events, median of --repeat after one
set-up call), the set-up call, the device memory peak over the evaluation, and the bytes of the eval exchange heaps.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIG = {"rmat-1m": dict(n_layers=3, n_hidden=256), "reddit-shaped": dict(n_layers=4, n_hidden=256),
          "products-shaped": dict(n_layers=3, n_hidden=128), "small": dict(n_layers=3, n_hidden=64)}


def _args(g, shape, dtype):
    from pipegcn_b200.synthetic import SHAPES
    base = dict(model="graphsage", backend="nccl", dtype=dtype, n_linear=0, n_feat=g.n_feat,
                n_class=SHAPES[shape]["n_class"], n_train=int(g.train_mask.sum()), dropout=0.5, norm="layer", lr=1e-2,
                weight_decay=0.0, use_pp=False, enable_pipeline=True, feat_corr=False, grad_corr=False,
                corr_momentum=0.95, seed=0, n_epochs=1, log_every=1, **CONFIG.get(shape, CONFIG["small"]))
    return argparse.Namespace(**base)


def _time(fn, repeat):
    first0, first1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    first0.record()
    fn()
    first1.record()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    ms.sort()
    return first0.elapsed_time(first1), ms[len(ms) // 2]


def _rank0(g, model, dtype, repeat):
    """--eval today: the whole graph built a second time on rank 0, the eval branch over all N rows."""
    from pipegcn_b200.evaluate import EvalSet, _logits, calc_acc
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    es = EvalSet(g, "cuda", dtype=dtype)
    held = torch.cuda.memory_allocated() - before

    def once():
        z = _logits(model, es.val)
        m, t = es.val["val_mask"], es.val["test_mask"]
        return calc_acc(z[m], es.val["label"][m]), calc_acc(z[t], es.val["label"][t])
    setup, ms = _time(once, repeat)
    peak = torch.cuda.max_memory_allocated()
    acc = once()
    del es
    return dict(ms=ms, first_ms=setup, peak_gb=peak / 1e9, eval_state_gb=held / 1e9, eval_heap_bytes=0, acc=acc)


def _partitioned(evaluate, heap_bytes, repeat):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    setup, ms = _time(evaluate, repeat)
    return dict(ms=ms, first_ms=setup, peak_gb=torch.cuda.max_memory_allocated() / 1e9, eval_heap_bytes=heap_bytes(),
                acc=evaluate())


def one_gpu(a):
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import LocalTrainer
    from pipegcn_b200.world import LocalWorld
    for shape in a.shapes:
        g = make_graph(shape, device="cuda")
        for P in a.parts:
            layouts = build_layouts(g, random_partition(g.n_nodes, P, device="cuda"), P)
            args = _args(g, shape, a.dtype)
            tr = LocalTrainer(layouts, args, LocalWorld(P, "cuda"))
            del layouts
            tr.run_epoch()
            torch.cuda.synchronize()
            res = _partitioned(tr.evaluate, lambda: sum(e.eval_heap_bytes for e in tr.engines), a.repeat)
            print(json.dumps(dict(shape=shape, path="partitioned", world="LocalWorld", P=P, dtype=a.dtype,
                                  gpu=torch.cuda.get_device_name(), **res)), flush=True)
            tr.release_eval()
            if P == a.parts[0]:
                res = _rank0(g, tr.engines[0].model, tr.engines[0].dtype, a.repeat)
                print(json.dumps(dict(shape=shape, path="rank0", world="LocalWorld", P=P, dtype=a.dtype,
                                      gpu=torch.cuda.get_device_name(), **res)), flush=True)
            del tr
            torch.cuda.empty_cache()
        del g
        torch.cuda.empty_cache()


def multi_gpu(a):
    import torch.distributed as dist
    from pipegcn_b200.partition import build_layouts
    from pipegcn_b200.synthetic import make_graph, random_partition
    from pipegcn_b200.train import RankEngine
    from pipegcn_b200.world import DistWorld
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    P = dist.get_world_size()
    for shape in a.shapes:
        g = make_graph(shape, device="cuda")
        lay = build_layouts(g, random_partition(g.n_nodes, P, device="cuda"), P, ranks=[rank])[0]
        args = _args(g, shape, a.dtype)
        if rank != 0:
            del g
        eng = RankEngine(lay, args, DistWorld())
        del lay
        eng.run_epoch()
        torch.cuda.synchronize()
        res = _partitioned(eng.evaluate, lambda: eng.eval_heap_bytes, a.repeat)
        if rank == 0:
            print(json.dumps(dict(shape=shape, path="partitioned", world="DistWorld", P=P, dtype=a.dtype,
                                  gpu=torch.cuda.get_device_name(), **res)), flush=True)
        eng.release_eval()
        if rank == 0:
            res = _rank0(g, eng.model, eng.dtype, a.repeat)
            print(json.dumps(dict(shape=shape, path="rank0", world="DistWorld", P=P, dtype=a.dtype,
                                  gpu=torch.cuda.get_device_name(), **res)), flush=True)
            del g
        dist.barrier()
        eng.buffer.release()
        del eng
        torch.cuda.empty_cache()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["rmat-1m", "reddit-shaped"])
    ap.add_argument("--parts", nargs="+", type=int, default=[1, 4])
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--dtype", default="bf16", choices=["fp32", "bf16"])
    a = ap.parse_args()
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        multi_gpu(a)
    else:
        one_gpu(a)


if __name__ == "__main__":
    main()
