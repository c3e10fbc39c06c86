"""Launcher: one process per partition / GPU (entry point of PipeGCN/main.py).

    python main.py --dataset synthetic:rmat-1m --n-partitions 4 --n-layers 3 --n-hidden 256 \
        --enable-pipeline --dtype bf16 --partition-method random --no-eval --fix-seed
"""
import os
import random
import warnings

import torch
import torch.multiprocessing as mp

from pipegcn_b200 import train
from pipegcn_b200.helper.parser import create_parser

if __name__ == '__main__':
    args = create_parser()
    if not args.fix_seed:
        if args.parts_per_node < args.n_partitions:
            warnings.warn('Please enable `--fix-seed` for multi-node training.')
        args.seed = random.randint(0, 1 << 31)
    if args.graph_name == '':
        args.graph_name = '%s-%d-%s-%s-%s' % (args.dataset, args.n_partitions, args.partition_method,
                                              args.partition_obj, 'induc' if args.inductive else 'trans')
    print(args)
    if args.backend not in ('nccl', 'nvlink'):
        # the reference raises for everything but gloo (main.py:60-65); this engine is NVLink/NCCL only
        raise NotImplementedError("backend '%s'" % args.backend)
    n_dev = torch.cuda.device_count()
    if n_dev < min(args.parts_per_node, args.n_partitions):
        raise RuntimeError('one GPU per partition is required: %d partitions, %d GPUs' % (args.n_partitions, n_dev))
    mp.set_start_method('spawn', force=True)
    start = args.node_rank * args.parts_per_node
    procs = []
    for i in range(start, min(start + args.parts_per_node, args.n_partitions)):
        p = mp.Process(target=train.init_processes, args=(i, args.n_partitions, args))
        p.start()
        procs.append(p)
    for p in procs:
        p.join()
