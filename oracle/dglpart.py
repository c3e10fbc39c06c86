"""Oracle: what `dgl.distributed.partition_graph` + `load_partition` hand to `train.run`.

TEST INFRASTRUCTURE (see oracle/__init__.py).  DGL is a third-party dependency
absent from PipeGCN (fork `chwan-rice/dgl`, unpinned HEAD,
PipeGCN/setup.sh:3); its documented behaviour for the call at
PipeGCN/helper/utils.py:143-144 (`reshuffle=True, balance_edges=False`,
default 1-hop halo) is restated here:

* nodes of partition p get the contiguous global id range
  [start_p, start_p + n_p), ascending original id inside a partition;
* the partition subgraph lists the inner nodes first (local id = global id -
  start_p) followed by the halo nodes (1-hop in-neighbours owned elsewhere);
* its edges are all in-edges of inner nodes;
* `ndata[dgl.NID]` = reshuffled global ids, `ndata['part_id']` = owner of every
  node, `ndata['inner_node']` = 1 for inner nodes;
* node features (`feat`, `label`, `in_degree`, `train_mask`) cover inner nodes
  only (PipeGCN/helper/utils.py:105-123).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import torch

NID = "_ID"   # value of dgl.NID


class GraphPartitionBook:
    """`gpb.partid2nids(i)` (used at PipeGCN/train.py:91-92,127; utils.py:171)."""

    def __init__(self, starts: torch.Tensor):
        self._starts = starts

    def partid2nids(self, i: int) -> torch.Tensor:
        return torch.arange(int(self._starts[i]), int(self._starts[i + 1]), dtype=torch.int64)


@dataclass
class DglPartition:
    su: torch.Tensor              # subgraph edge sources (subgraph node ids)
    sv: torch.Tensor              # subgraph edge destinations (always inner)
    n_nodes: int                  # inner + halo
    node_dict: Dict[str, torch.Tensor]
    gpb: GraphPartitionBook


def partition_graph(n_nodes: int, src: torch.Tensor, dst: torch.Tensor, part: torch.Tensor, n_parts: int,
                    feat: torch.Tensor, label: torch.Tensor, train_mask: torch.Tensor) -> List[DglPartition]:
    part = part.to(torch.int64)
    order = torch.argsort(part, stable=True)
    counts = torch.bincount(part, minlength=n_parts)
    starts = torch.zeros(n_parts + 1, dtype=torch.int64)
    starts[1:] = torch.cumsum(counts, 0)
    new_gid = torch.empty(n_nodes, dtype=torch.int64)
    new_gid[order] = torch.arange(n_nodes, dtype=torch.int64)
    in_degree = torch.bincount(dst, minlength=n_nodes)            # g.in_degrees(), utils.py:142
    gs, gd = new_gid[src], new_gid[dst]                            # edges in reshuffled ids
    owner_of_new = part[order]                                     # owner of reshuffled id
    gpb = GraphPartitionBook(starts)
    out = []
    for p in range(n_parts):
        lo, hi = int(starts[p]), int(starts[p + 1])
        em = (gd >= lo) & (gd < hi)
        es, ed = gs[em], gd[em]
        halo = torch.unique(es[(es < lo) | (es >= hi)])            # ascending global id
        nodes = torch.cat([torch.arange(lo, hi, dtype=torch.int64), halo])
        lookup = torch.full((n_nodes,), -1, dtype=torch.int64)
        lookup[nodes] = torch.arange(nodes.numel(), dtype=torch.int64)
        inner_orig = order[lo:hi]
        node_dict = {
            NID: nodes,
            "part_id": owner_of_new[nodes],
            "inner_node": (torch.arange(nodes.numel()) < (hi - lo)),
            "feat": feat[inner_orig].clone(),
            "label": label[inner_orig].clone(),
            "in_degree": in_degree[inner_orig].clone(),
            "train_mask": train_mask[inner_orig].clone().bool(),
        }
        out.append(DglPartition(lookup[es], lookup[ed], int(nodes.numel()), node_dict, gpb))
    return out
