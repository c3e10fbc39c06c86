"""Oracle: per-process set-up of the halo index space (SURVEY.md §8a rows S1-S4).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates, on plain host tensors
and for all ranks of a simulated world at once:

  get_boundary      PipeGCN/helper/utils.py:154-188
  get_pos           PipeGCN/train.py:84-98
  create_inner_graphPipeGCN/train.py:113-117
  order_graph       PipeGCN/train.py:120-131
  construct         PipeGCN/train.py:206-229
  move_train_first  PipeGCN/train.py:134-155
  get_recv_shape    PipeGCN/train.py:101-110
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from .dglpart import NID, DglPartition


@dataclass
class RankSetup:
    rank: int
    size: int
    num_in: int
    num_all: int
    u: torch.Tensor                       # bipartite `_U` -> `_V` edges, int64
    v: torch.Tensor
    in_deg: torch.Tensor                  # [num_in] int64
    boundary: List[Optional[torch.Tensor]]
    recv_shape: List[Optional[int]]
    node_dict: Dict[str, torch.Tensor]    # feat / label / train_mask / in_degree of inner nodes


def get_boundary(parts: List[DglPartition]) -> List[List[Optional[torch.Tensor]]]:
    """utils.py:154-188: rank `right` receives, sorted, the owner-local ids that `rank` borrows from it."""
    size = len(parts)
    boundary = [[None] * size for _ in range(size)]
    for rank, p in enumerate(parts):
        nd = p.node_dict
        for right in range(size):
            if right == rank:
                continue
            belong_right = nd["part_id"] == right                      # utils.py:162
            start = int(p.gpb.partid2nids(right)[0]) if p.gpb.partid2nids(right).numel() else 0
            v = nd[NID][belong_right] - start                          # utils.py:171-172
            boundary[right][rank], _ = torch.sort(v)                   # utils.py:181 (on the receiver)
    return boundary


def get_pos(p: DglPartition, rank: int, size: int):
    """train.py:84-98: owner-local id -> my subgraph node id, per peer."""
    pos = []
    nd = p.node_dict
    for i in range(size):
        if i == rank:
            pos.append(None)
            continue
        ids = p.gpb.partid2nids(i)
        start = int(ids[0]) if ids.numel() else 0
        q = torch.full((ids.numel(),), -1, dtype=torch.int64)
        in_idx = torch.nonzero(nd["part_id"] == i, as_tuple=True)[0]
        q[nd[NID][in_idx] - start] = in_idx
        pos.append(q)
    return pos


def _out_edges(su, sv, n_nodes, nodes):
    """DGL `graph.out_edges(nodes)` / `out_degrees(nodes)`: edges grouped by node, in the order of `nodes`."""
    order = torch.argsort(su, stable=True)
    counts = torch.bincount(su, minlength=n_nodes)
    ptr = torch.zeros(n_nodes + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(counts, 0)
    deg = counts[nodes]
    rep = torch.repeat_interleave(torch.arange(nodes.numel()), deg)
    offs = torch.arange(int(deg.sum())) - torch.repeat_interleave(torch.cumsum(deg, 0) - deg, deg)
    eids = order[ptr[nodes][rep] + offs]
    return deg, sv[eids]


def construct(p: DglPartition, rank: int, size: int, pos, one_hops):
    """train.py:113-117 (inner graph) + 206-229: `_U` = [inner | halo of peer 0 | peer 1 | ...]."""
    inner = p.node_dict["inner_node"].bool()
    sel = inner[p.su] & inner[p.sv]                                    # train.py:115
    tot = int(inner.sum())                                             # part.num_nodes()
    u_list, v_list = [p.su[sel]], [p.sv[sel]]
    for i in range(size):
        if i == rank:
            continue
        u = one_hops[i]
        if u.shape[0] == 0:
            continue
        u = pos[i][u]                                                  # train.py:218
        deg, v = _out_edges(p.su, p.sv, p.n_nodes, u)                  # train.py:219,221
        u_ = torch.repeat_interleave(torch.arange(u.shape[0]), deg) + tot
        tot += u.shape[0]
        u_list.append(u_)
        v_list.append(v)
    return torch.cat(u_list), torch.cat(v_list), tot


def order_graph(p: DglPartition, rank: int, size: int, pos):
    """train.py:120-131: halo of peer i ordered by i's local id."""
    nd = p.node_dict
    one_hops = []
    for i in range(size):
        if i == rank:
            one_hops.append(None)
            continue
        ids = p.gpb.partid2nids(i)
        start = int(ids[0]) if ids.numel() else 0
        nodes = nd[NID][nd["part_id"] == i] - start
        nodes, _ = torch.sort(nodes)
        one_hops.append(nodes)
    return construct(p, rank, size, pos, one_hops)


def move_train_first(u, v, num_tot, node_dict, boundary):
    """train.py:134-155."""
    train_mask = node_dict["train_mask"]
    num_train = int(torch.count_nonzero(train_mask))
    new_id = torch.zeros(num_tot, dtype=torch.int64)
    new_id[train_mask] = torch.arange(num_train)
    new_id[~train_mask] = torch.arange(num_train, num_tot)
    u = u.clone()
    m = u < num_tot
    u[m] = new_id[u[m]]                                                # train.py:144
    v = new_id[v]                                                      # train.py:145
    out = {}
    for key in ("feat", "label", "in_degree", "train_mask"):           # inner-node rows (train.py:148-149)
        t = node_dict[key].clone()
        t[new_id] = node_dict[key][0:num_tot].clone()
        out[key] = t
    boundary = [None if b is None else new_id[b] for b in boundary]    # train.py:151-153
    return u, v, out, boundary


def get_recv_shape(p: DglPartition, rank: int, size: int):
    """train.py:101-110."""
    return [None if i == rank else int((p.node_dict["part_id"] == i).sum()) for i in range(size)]


def setup_world(parts: List[DglPartition]) -> List[RankSetup]:
    """The part of `train.run` before `init_buffer` (train.py:262-281) for every rank."""
    size = len(parts)
    boundary_all = get_boundary(parts)
    out = []
    for rank, p in enumerate(parts):
        num_in = int(p.node_dict["inner_node"].bool().sum())          # train.py:263
        pos = get_pos(p, rank, size)
        u, v, num_all = order_graph(p, rank, size, pos)
        u, v, nd, boundary = move_train_first(u, v, num_in, p.node_dict, boundary_all[rank])
        out.append(RankSetup(rank, size, num_in, num_all, u, v, nd["in_degree"], boundary,
                             get_recv_shape(p, rank, size), nd))
    return out


def precompute(setups: List[RankSetup]) -> List[torch.Tensor]:
    """`--use-pp` (train.py:169-189 with data_transfer / merge_feature, utils.py:191-223): one exchange of the raw
    boundary features, neighbour mean over the `_U` graph, feat <- cat(feat, mean) [N_in, 2 * n_feat]."""
    size = len(setups)
    out = []
    for r, s in enumerate(setups):
        feat = s.node_dict["feat"]
        recv = [setups[j].node_dict["feat"][setups[j].boundary[r]] for j in range(size) if j != r]   # ascending peers
        merged = torch.cat([feat] + recv)                                   # merge_feature, utils.py:216-223
        summed = torch.zeros(s.num_in, feat.shape[1]).index_add_(0, s.v, merged[s.u])
        mean = summed / s.in_deg[0:s.num_in].unsqueeze(1)                   # train.py:186
        out.append(torch.cat([feat, mean[0:s.num_in]], dim=1))              # train.py:187
    return out
