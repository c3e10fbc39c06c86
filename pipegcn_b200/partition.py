"""Per-partition index spaces of the hot path (SURVEY.md §8a rows S1-S4, Appendix A).

The reference derives these per process from a DGL partition through
`get_boundary` (PipeGCN/helper/utils.py:154-188), `get_pos`
(PipeGCN/train.py:84-98), `order_graph`/`construct` (train.py:120-131,
206-229), `move_train_first` (train.py:134-155) and `get_recv_shape`
(train.py:101-110).  Here the same layouts are produced in one vectorised pass
over the global edge list (torch, host or GPU), without DGL:

* global reshuffle: nodes of partition p get a contiguous id range, ascending
  original id inside a partition (DGL `reshuffle=True`, utils.py:143-144);
* `_U` (source) space of rank r: [inner | halo of peer 0 | halo of peer 1 ...],
  halo of peer j ordered by j's local id (train.py:129, 211-223);
* `boundary[j]`: r's inner rows peer j holds as halo, in the order of j's halo
  list (== ascending r-local id before `move_train_first`, utils.py:181);
* `move_train_first`: inner ids relabelled so train rows come first, applied to
  rows, inner sources and boundary lists alike (train.py:139-153).

The result carries the adjacency twice: CSR by destination (forward aggregate)
and CSC by source over the whole `_U` space (backward aggregate), int32 like the
reference's on-GPU ids (train.py:78-79).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import torch

from .synthetic import GlobalGraph


@dataclass
class PartitionLayout:
    rank: int
    size: int
    num_in: int                      # N_in: inner (owned) rows == number of `_V` nodes
    num_all: int                     # N_in + H: number of `_U` nodes
    indptr: torch.Tensor             # [N_in+1] int32, CSR by destination
    indices: torch.Tensor            # [nnz]    int32, source ids in [0, num_all)
    t_indptr: torch.Tensor           # [num_all+1] int32, CSC by source
    t_indices: torch.Tensor          # [nnz]    int32, destination ids in [0, N_in)
    in_deg: torch.Tensor             # [N_in] int64, GLOBAL in-degree incl. self loop (utils.py:142)
    boundary: List[Optional[torch.Tensor]]   # per peer: int64 inner row ids to send (None for self)
    recv_shape: List[Optional[int]]          # per peer: H_j (None for self)
    feat: torch.Tensor               # [N_in, F]
    label: torch.Tensor              # [N_in]
    train_mask: torch.Tensor         # [N_in] bool (first n_train_local entries True)
    inner_gid: torch.Tensor          # [N_in] original global id of every inner row (after permutation)
    halo_gid: torch.Tensor           # [H] original global id of every halo row
    n_train_global: int = 0
    extra: dict = field(default_factory=dict)
    # [N_in] bool, same row order as `label`: the evaluation masks of the inner rows (GlobalGraph.val_mask /
    # test_mask through inner_gid); None when the builder did not provide them
    val_mask: Optional[torch.Tensor] = None
    test_mask: Optional[torch.Tensor] = None

    @property
    def nnz(self) -> int:
        return int(self.indices.numel())

    @property
    def n_train_local(self) -> int:
        return int(self.train_mask.sum().item())

    def to(self, device) -> "PartitionLayout":
        def mv(x):
            return x.to(device) if isinstance(x, torch.Tensor) else x
        kw = {k: mv(v) for k, v in self.__dict__.items() if k not in ("boundary", "extra")}
        kw["boundary"] = [mv(b) for b in self.boundary]
        kw["extra"] = dict(self.extra)
        return PartitionLayout(**kw)


def _csr_from_pairs(rows: torch.Tensor, cols: torch.Tensor, n_rows: int, n_cols: int):
    """Sort (row, col) pairs and return int32 (indptr, indices), columns ascending in a row."""
    key = rows * max(n_cols, 1) + cols
    order = torch.argsort(key)
    cols_sorted = cols[order].to(torch.int32)
    counts = torch.bincount(rows, minlength=n_rows)
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=rows.device)
    indptr[1:] = torch.cumsum(counts, 0)
    return indptr.to(torch.int32), cols_sorted


class PartitionPlan:
    """Global pass shared by all ranks: reshuffled ids and the cross-partition halo table."""

    def __init__(self, g: GlobalGraph, part: torch.Tensor, n_parts: int):
        self.g = g
        self.P = int(n_parts)
        dev = g.src.device
        part = part.to(dev).to(torch.int64)
        self.part = part
        n = g.n_nodes
        order = torch.argsort(part, stable=True)            # ascending original id inside a part
        counts = torch.bincount(part, minlength=self.P)
        self.part_count = counts
        self.part_start = torch.zeros(self.P + 1, dtype=torch.int64, device=dev)
        self.part_start[1:] = torch.cumsum(counts, 0)
        new_gid = torch.empty(n, dtype=torch.int64, device=dev)
        new_gid[order] = torch.arange(n, dtype=torch.int64, device=dev)
        self.local_id = new_gid - self.part_start[part]     # owner-local id of every node
        self.order = order                                   # order[p_start + l] = original id
        self.in_deg = g.in_degrees()
        self.n_max = int(counts.max().item()) if n > 0 else 1
        # cross-partition (dst part j, src part r, src local id) triples, unique & sorted:
        sp, dp = part[g.src], part[g.dst]
        cross = sp != dp
        key = (dp[cross] * self.P + sp[cross]) * self.n_max + self.local_id[g.src[cross]]
        self.cross_key = torch.unique(key)                   # sorted ascending
        pair = self.cross_key // self.n_max
        self.pair_count = torch.bincount(pair, minlength=self.P * self.P)  # [j*P + r] = |halo of j owned by r|
        self.pair_start = torch.zeros(self.P * self.P + 1, dtype=torch.int64, device=dev)
        self.pair_start[1:] = torch.cumsum(self.pair_count, 0)
        self.n_train_global = int(g.train_mask.sum().item())

    def halo_list(self, holder: int, owner: int) -> torch.Tensor:
        """Owner-local ids (ascending) of the rows `holder` borrows from `owner`."""
        k = holder * self.P + owner
        lo, hi = int(self.pair_start[k].item()), int(self.pair_start[k + 1].item())
        return self.cross_key[lo:hi] % self.n_max

    def build(self, rank: int) -> PartitionLayout:
        g, P, part = self.g, self.P, self.part
        dev = g.src.device
        r = int(rank)
        n_in = int(self.part_count[r].item())
        inner_orig = self.order[int(self.part_start[r].item()): int(self.part_start[r + 1].item())]

        # ---- move_train_first relabelling of inner ids (train.py:139-141)
        tm = g.train_mask[inner_orig]
        n_train = int(tm.sum().item())
        new_id = torch.empty(n_in, dtype=torch.int64, device=dev)
        new_id[tm] = torch.arange(n_train, dtype=torch.int64, device=dev)
        new_id[~tm] = torch.arange(n_train, n_in, dtype=torch.int64, device=dev)

        # ---- edges whose destination is owned by r
        emask = part[g.dst] == r
        es, ed = g.src[emask], g.dst[emask]
        v = new_id[self.local_id[ed]]
        owner = part[es]
        is_inner = owner == r
        u = torch.empty_like(es)
        u[is_inner] = new_id[self.local_id[es[is_inner]]]
        # halo rows: ascending (owner, owner-local id) == [peer 0 | peer 1 | ...] (train.py:211-223)
        hkey = owner[~is_inner] * self.n_max + self.local_id[es[~is_inner]]
        hsorted, hinv = torch.unique(hkey, return_inverse=True)
        u[~is_inner] = n_in + hinv
        n_halo = int(hsorted.numel())
        howner = hsorted // self.n_max
        recv_cnt = torch.bincount(howner, minlength=P)
        recv_shape: List[Optional[int]] = [None if j == r else int(recv_cnt[j].item()) for j in range(P)]
        halo_gid = self.order[self.part_start[howner] + hsorted % self.n_max]
        num_all = n_in + n_halo

        indptr, indices = _csr_from_pairs(v, u, n_in, num_all)
        t_indptr, t_indices = _csr_from_pairs(u, v, num_all, n_in)

        # ---- boundary lists: rows of r that peer j holds as halo (utils.py:154-188), relabelled
        boundary: List[Optional[torch.Tensor]] = []
        for j in range(P):
            boundary.append(None if j == r else new_id[self.halo_list(j, r)])

        def permute_rows(x):
            out = torch.empty_like(x)
            out[new_id] = x                 # node_dict[key][new_id] = node_dict[key].clone() (train.py:149)
            return out

        inner_gid = permute_rows(inner_orig)
        return PartitionLayout(
            rank=r, size=P, num_in=n_in, num_all=num_all,
            indptr=indptr, indices=indices, t_indptr=t_indptr, t_indices=t_indices,
            in_deg=self.in_deg[inner_gid], boundary=boundary, recv_shape=recv_shape,
            feat=g.feat[inner_gid], label=g.label[inner_gid], train_mask=g.train_mask[inner_gid],
            inner_gid=inner_gid, halo_gid=halo_gid, n_train_global=self.n_train_global,
            val_mask=g.val_mask[inner_gid], test_mask=g.test_mask[inner_gid])


def build_layouts(g: GlobalGraph, part: torch.Tensor, n_parts: int, ranks=None) -> List[PartitionLayout]:
    plan = PartitionPlan(g, part, n_parts)
    ranks = range(n_parts) if ranks is None else ranks
    return [plan.build(r) for r in ranks]


def extend_partition(train_mask: torch.Tensor, train_part: torch.Tensor, n_parts: int, seed: int = 2) -> torch.Tensor:
    """Node -> partition of the whole graph for the --inductive evaluation graphs: the training nodes keep the part
    of the training partition (`train_part`, in ascending id order of the training nodes), every other node gets a
    seeded uniform draw -- the same on every rank."""
    from .synthetic import random_partition
    part = random_partition(int(train_mask.numel()), n_parts, seed=seed, device=train_mask.device)
    part[train_mask] = train_part.to(part.device).to(part.dtype)
    return part


def build_eval_layout(g: GlobalGraph, keep: Optional[torch.Tensor], part: torch.Tensor, n_parts: int,
                      rank: int) -> PartitionLayout:
    """Rank `rank`'s layout of the subgraph of `g` induced by `keep` (None: all of g) under the node -> partition map
    `part` of g.  Ids (inner_gid, halo_gid) are those of the subgraph; val_mask / test_mask follow g's rule."""
    from .synthetic import induced_subgraph
    if keep is None:
        sub, ids = g, None
    else:
        sub, ids = induced_subgraph(g, keep)
    lay = PartitionPlan(sub, part if ids is None else part[ids], n_parts).build(rank)
    gid = lay.inner_gid if ids is None else ids[lay.inner_gid]
    lay.val_mask, lay.test_mask = g.val_mask[gid], g.test_mask[gid]
    return lay


def get_layer_size(n_feat: int, n_hidden: int, n_class: int, n_layers: int) -> List[int]:
    """[n_feat, h, ..., h, n_class] with n_layers+1 entries (PipeGCN/helper/utils.py:147-151)."""
    return [n_feat] + [n_hidden] * (n_layers - 1) + [n_class]
