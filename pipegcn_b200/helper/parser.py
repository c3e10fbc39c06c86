"""Command line of the trainer: the flags of PipeGCN/helper/parser.py:8-69.

Same names, aliases and defaults, with three deliberate differences: `--backend`
defaults to `nccl` (the reference implements gloo only; this engine implements the
NVLink/NCCL path only), `--dataset` also accepts `synthetic:<shape>` (shapes in
pipegcn_b200/synthetic.py), `--model` accepts `gcn` as an alias of `graphsage`, and
`--dtype {fp32,bf16}` selects the activation storage type.

`--eval-partitioned` (off by default; not in the reference) makes `--eval` partition-parallel: every rank evaluates
its own inner rows over an exact halo exchange and the accuracy counts are summed across ranks, instead of rank 0
evaluating the whole graph, which it would have to hold a second time.  The printed lines, the result file and the
checkpoint keep their formats.  When the flag is absent the namespace has no `eval_partitioned` attribute (read it
with getattr(args, 'eval_partitioned', False)), so the parsed flags stay the reference's.

`--sampling-rate p` (0 < p <= 1; not in the reference) turns on boundary-node sampling (BNS-GCN) in synchronous
training: every epoch each partition keeps a random fraction p of its halo nodes and drops the rest from its graph for
that epoch, so the halo exchange moves p times the bytes.  Evaluation always uses the full graph.  Like
`--eval-partitioned` it has a suppressed default: read it with getattr(args, 'sampling_rate', 1.0).
"""
import argparse

# (flag, alias-with-underscores?, kwargs)
_FLAGS = [
    ("dataset", dict(type=str, default='reddit', help="the input dataset (or synthetic:<shape>)")),
    ("graph-name", dict(type=str, default='')),
    ("model", dict(type=str, default='graphsage', help="model for training (graphsage | gcn)")),
    ("dropout", dict(type=float, default=0.5, help="dropout probability")),
    ("lr", dict(type=float, default=1e-2, help="learning rate")),
    ("n-epochs", dict(type=int, default=200, help="the number of training epochs")),
    ("n-partitions", dict(type=int, default=2, help="the number of partitions")),
    ("n-hidden", dict(type=int, default=16, help="the number of hidden units")),
    ("n-layers", dict(type=int, default=2, help="the number of GCN layers")),
    ("n-linear", dict(type=int, default=0, help="the number of linear layers")),
    ("norm", dict(choices=['layer', 'batch'], default='layer', help="normalization method")),
    ("weight-decay", dict(type=float, default=0, help="weight for L2 loss")),
    ("n-feat", dict(type=int, default=0)),
    ("n-class", dict(type=int, default=0)),
    ("n-train", dict(type=int, default=0)),
    ("skip-partition", dict(action='store_true', help="skip graph partition")),
    ("partition-obj", dict(choices=['vol', 'cut'], default='vol', help="partition objective function")),
    ("partition-method", dict(choices=['metis', 'random'], default='metis', help="graph partition method")),
    ("enable-pipeline", dict(action='store_true')),
    ("feat-corr", dict(action='store_true')),
    ("grad-corr", dict(action='store_true')),
    ("corr-momentum", dict(type=float, default=0.95)),
    ("use-pp", dict(action='store_true', help="whether to use precomputation")),
    ("inductive", dict(action='store_true', help="inductive learning setting")),
    ("fix-seed", dict(action='store_true', help="fix random seed")),
    ("seed", dict(type=int, default=0)),
    ("log-every", dict(type=int, default=10)),
    ("backend", dict(type=str, default='nccl')),
    ("port", dict(type=int, default=18118, help="the network port for communication")),
    ("master-addr", dict(type=str, default="127.0.0.1")),
    ("node-rank", dict(type=int, default=0)),
    ("parts-per-node", dict(type=int, default=10)),
    ("dtype", dict(choices=['fp32', 'bf16'], default='fp32', help="activation storage type")),
]


def _sampling_rate(text):
    try:
        p = float(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid sampling rate '{text}'")
    if not 0.0 < p <= 1.0:           # also refuses nan
        raise argparse.ArgumentTypeError(f"sampling rate {text}: expected 0 < p <= 1")
    return p


def build_parser():
    parser = argparse.ArgumentParser(description='PipeGCN on H100')
    for flag, kw in _FLAGS:
        names = ["--" + flag]
        if "-" in flag:
            names.append("--" + flag.replace("-", "_"))
        parser.add_argument(*names, **kw)
    parser.add_argument('--eval', action='store_true', help="enable evaluation")
    parser.add_argument('--no-eval', action='store_false', dest='eval', help="disable evaluation")
    parser.set_defaults(eval=True)
    parser.add_argument('--no-partition-cache', action='store_false', dest='partition_cache',
                        help="do not read/write partitions/<graph_name>/part.pt")
    parser.set_defaults(partition_cache=True)
    parser.add_argument('--eval-partitioned', '--eval_partitioned', action='store_true', default=argparse.SUPPRESS,
                        help="with --eval: every rank evaluates its own nodes (exact halo exchange) instead of rank 0 "
                             "evaluating the whole graph")
    parser.add_argument('--sampling-rate', '--sampling_rate', type=_sampling_rate, default=argparse.SUPPRESS,
                        help="boundary-node sampling: the fraction of halo nodes every partition keeps per epoch "
                             "(synchronous training; default 1 = all)")
    return parser


def create_parser(argv=None):
    return build_parser().parse_args(argv)
