"""CPU oracle of the PipeGCN hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain-torch (CPU, fp32) restatement of the reference algorithm for the path
BASELINE.json's `north_star` names (SURVEY.md §8): the halo feature/gradient
exchange with one-epoch staleness and EMA correction
(PipeGCN/helper/feature_buffer.py), the GraphSAGE-mean layer
(PipeGCN/module/layer.py), the model loop (PipeGCN/module/model.py),
the gradient reducer (PipeGCN/helper/reducer.py) and the per-process
set-up / epoch loop of PipeGCN/train.py.  Every function cites the
reference file:line it follows.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s `cpu_baseline` /
`--impl reference` legs may import this package, and only as the checker or the
timed CPU baseline.  Nothing under `pipegcn_b200/` imports it.

Third-party arithmetic that is NOT under PipeGCN and is restated here
from its documented behaviour: DGL 0.8 (fork `chwan-rice/dgl`, unpinned --
PipeGCN/setup.sh:3 clones HEAD): `update_all(copy_src, sum)` == 0/1 CSR
`A @ X`; `partition_graph(reshuffle=True)` node/halo conventions
(oracle/dglpart.py).

Pinning: the reference ships no tests, golden vectors or fixtures (SURVEY.md
§4).  The oracle is pinned against outputs of the UNMODIFIED reference modules
(`helper/feature_buffer.py`, `module/layer.py`, `module/model.py`,
`helper/reducer.py`, the set-up helpers of `train.py`/`helper/utils.py`)
executed on a host over gloo with CUDA calls redirected to the host
and a minimal stand-in for the absent DGL graph container; the script is
`tests/golden/make_golden.py`, its outputs are the fixtures in `tests/golden/`.
"""
