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

`--model gat` trains graph attention (DGL's GATConv) instead of GraphSAGE, `--model gatv2` dynamic graph attention
(DGL's GATv2Conv) and `--model transformer` the graph transformer (PyG's TransformerConv: dot-product attention over
the in-edges with a skip connection); `--n-heads k` (not in the reference, default 4, suppressed like
`--sampling-rate`: read it with getattr(args, 'n_heads', 4)) sets the heads per hidden layer of each of them.

`--model graphconv` (not in the reference) trains Kipf & Welling's graph convolution (DGL's GraphConv, norm='both'):
every layer aggregates c_v sum_u c_u h_u with c = deg^-1/2, the halo rows' degrees supplied by their owners.  `--model
gcn` stays the reference's name for GraphSAGE.  It cannot be combined with --aggregator pool or --sampling-rate < 1.

`--halo-bits b` (8 or 4; not in the reference) quantises the per-epoch halo messages of graph layers >= 1, features
forward and gradients backward: every row travels as b-bit codes with an fp32 (lo, scale), stochastically rounded so
the message stays unbiased, and the receiver decodes it before anything reads it.  Layer 0, --use-pp and the
evaluation exchange stay exact; it cannot be combined with --sampling-rate p < 1.  Suppressed like `--sampling-rate`:
read it with getattr(args, 'halo_bits', None).

`--aggregator {mean,pool}` (not in the reference) selects the neighbour reduction of the GraphSAGE layers: `mean` (the
reference's) or `pool`, Hamilton et al.'s max-pool aggregator (DGL `SAGEConv(aggregator_type='pool')`): every layer
takes the element-wise neighbour maximum of ReLU(h Wp^T + bp).  It cannot be combined with --model gat, gatv2 or
transformer, or with --use-pp.
Suppressed like `--sampling-rate`: read it with getattr(args, 'aggregator', 'mean').

`--model gcnii` (not in the reference) trains GCNII (Chen et al., ICML 2020; DGL's GCN2Conv): graph layer 0 is a linear
fc_in in front of its convolution, every convolution adds alpha times the initial representation h0 to its scaled
aggregate and maps it through (1 - beta_l) I + beta_l W1 with beta_l = ln(lambda / l + 1).  `--n-layers` counts fc_in's
layer, the convolutions and the `--n-linear` (>= 1) trailing linears.  `--gcnii-alpha a` (0 <= a <= 1, default 0.1)
and `--gcnii-lambda l` (l > 0, finite, default 0.5) set alpha and lambda; suppressed like `--sampling-rate`: read them
with getattr(args, 'gcnii_alpha', 0.1) and getattr(args, 'gcnii_lambda', 0.5).  It cannot be combined with --use-pp,
--aggregator pool or --sampling-rate < 1.

`--model pna` (not in the reference) trains principal neighbourhood aggregation (Corso et al., NeurIPS 2020; DGL's
PNAConvTower): every layer reduces the messages M(cat(h_u, h_v)) with mean, max, min and std, scales the result by
the identity, log(D + 1) / delta and delta / log(D + 1) (D the in-degree, delta the mean of log(D + 1) over the
training graph, derived at set-up), and maps cat(h_v, the 12 scaled aggregates) through a linear U.  It has no flags
of its own.  It cannot be combined with --aggregator pool, --use-pp or --sampling-rate < 1.

`--model genconv` (not in the reference) trains the softmax-aggregation graph convolution of DeeperGCN (Li et al., 2020;
PyG's GENConv with aggr='softmax'): every layer aggregates m_u = ReLU(x_src[u]) + 1e-7 with a per-channel softmax of
t m_u over the in-edges, adds x_dst and maps the sum through a two-layer MLP [d, 2d, d].  `--genconv-t T` (a finite
float, default 1.0; 0 and negative values are allowed) sets the temperature, and `--genconv-learn-t` makes it a learnt
parameter (`aggr_module.t` of every graph layer).  Both are suppressed like `--sampling-rate`: read them with
getattr(args, 'genconv_t', 1.0) and getattr(args, 'genconv_learn_t', False).  It works with boundary-node sampling
and cannot be combined with --use-pp or --aggregator pool.

`--model resgatedgcn` (not in the reference) trains the residual gated graph convolution of Bresson & Laurent (2017;
PyG's ResGatedGraphConv): every layer sums the values val_u of its in-edges, each weighted by its own per-channel gate
sigmoid(k_v + q_u), and adds a skip linear of h_v and a bias.  It has no flags of its own (--n-heads is ignored).  It
works with boundary-node sampling and cannot be combined with --use-pp or --aggregator pool.

`--model monet` (not in the reference) trains the Gaussian mixture model convolution of MoNet (Monti et al., CVPR 2017;
DGL's GMMConv with the mean aggregator) on the degree pseudo-coordinates e_uv = (c_u, c_v), c = deg^-1/2 (the halo
rows' degrees supplied by their owners): every layer averages over the in-edges sum_k w_k(e_uv) h_u W_k^T, with K
Gaussian weights w_k of learnt means mu and inverse widths inv_sigma.  `--monet-kernels K` (an integer 1 <= K <= 8,
default 3) sets K; suppressed like `--sampling-rate`: read it with getattr(args, 'monet_kernels', 3).  --n-heads is
ignored.  It cannot be combined with --use-pp, --aggregator pool or --sampling-rate < 1.
"""
import argparse

# (flag, alias-with-underscores?, kwargs)
_FLAGS = [
    ("dataset", dict(type=str, default='reddit', help="the input dataset (or synthetic:<shape>)")),
    ("graph-name", dict(type=str, default='')),
    ("model", dict(type=str, default='graphsage', help="model for training (graphsage | gcn | gat | gatv2 | transformer | "
                                                              "graphconv | gcnii | pna | genconv | resgatedgcn | monet; "
                                                              "gcn is GraphSAGE)")),
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


def _n_heads(text):
    try:
        k = int(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid head count '{text}'")
    if k < 1:
        raise argparse.ArgumentTypeError(f"--n-heads {text}: expected a positive integer")
    return k


def _gcnii_alpha(text):
    try:
        a = float(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid GCNII alpha '{text}'")
    if not 0.0 <= a <= 1.0:          # also refuses nan
        raise argparse.ArgumentTypeError(f"--gcnii-alpha {text}: expected 0 <= alpha <= 1")
    return a


def _gcnii_lambda(text):
    try:
        lam = float(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid GCNII lambda '{text}'")
    if not 0.0 < lam < float('inf'):   # also refuses nan
        raise argparse.ArgumentTypeError(f"--gcnii-lambda {text}: expected a finite lambda > 0")
    return lam


def _genconv_t(text):
    try:
        t = float(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid GENConv temperature '{text}'")
    if not abs(t) < float('inf'):     # also refuses nan
        raise argparse.ArgumentTypeError(f"--genconv-t {text}: expected a finite temperature")
    return t


def _monet_kernels(text):
    try:
        k = int(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"invalid number of MoNet kernels '{text}'")
    if not 1 <= k <= 8:               # the kernel counts csrc/monet.cu is compiled for
        raise argparse.ArgumentTypeError(f"--monet-kernels {text}: expected 1 to 8 mixture kernels")
    return k


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
    parser.add_argument('--n-heads', '--n_heads', type=_n_heads, default=argparse.SUPPRESS,
                        help="--model gat / gatv2 / transformer: attention heads of every hidden layer "
                             "(default 4)")
    parser.add_argument('--halo-bits', '--halo_bits', type=int, choices=[8, 4], default=argparse.SUPPRESS,
                        help="send the halo messages of graph layers >= 1 as stochastically rounded 8- or 4-bit codes "
                             "(default: exact)")
    parser.add_argument('--aggregator', choices=['mean', 'pool'], default=argparse.SUPPRESS,
                        help="GraphSAGE neighbour aggregator: mean (default) or pool (max over ReLU(h Wp^T + bp))")
    parser.add_argument('--gcnii-alpha', '--gcnii_alpha', type=_gcnii_alpha, default=argparse.SUPPRESS,
                        help="--model gcnii: weight of the initial residual (0 <= alpha <= 1, default 0.1)")
    parser.add_argument('--gcnii-lambda', '--gcnii_lambda', type=_gcnii_lambda, default=argparse.SUPPRESS,
                        help="--model gcnii: beta_l = ln(lambda / l + 1) (lambda > 0, default 0.5)")
    parser.add_argument('--genconv-t', '--genconv_t', type=_genconv_t, default=argparse.SUPPRESS,
                        help="--model genconv: softmax temperature t (finite, default 1.0)")
    parser.add_argument('--genconv-learn-t', '--genconv_learn_t', action='store_true', default=argparse.SUPPRESS,
                        help="--model genconv: learn t (one scalar per graph layer, initialised to --genconv-t)")
    parser.add_argument('--monet-kernels', '--monet_kernels', type=_monet_kernels, default=argparse.SUPPRESS,
                        help="--model monet: Gaussian mixture kernels per layer (1 to 8, default 3)")
    return parser


def create_parser(argv=None):
    return build_parser().parse_args(argv)
