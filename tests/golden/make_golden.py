"""Generate the golden fixtures by running the UNMODIFIED reference (a checkout of GATECH-EIC/PipeGCN,
named by the environment variable PIPEGCN_REF) on the host.

    python tests/golden/make_golden.py            # writes tests/golden/ref_*.pt

One gloo process per partition, exactly like PipeGCN/main.py:51-57.  Every hot-path object is the
reference's own: `helper.context.buffer` (helper/feature_buffer.py), `module.model.GraphSAGE` /
`module.layer.GraphSAGELayer`, `helper.context.reducer` (helper/reducer.py), and the set-up helpers of train.py /
helper/utils.py (`create_inner_graph`, `move_to_cuda`, `get_boundary`, `get_pos`, `order_graph`, `construct`,
`move_train_first`, `get_recv_shape`, `get_layer_size`, `create_model`, `reduce_hook`).  Only what cannot exist
here is stood in for (tests/golden/ref_shims.py): CUDA streams/events/devices -> host no-ops, and the DGL graph
container.  The DGL *partitioner* output is produced by oracle/dglpart.py.  The epoch loop below repeats
PipeGCN/train.py:341-362 line by line so that per-layer tensors can be recorded.
"""
import argparse
import os
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["PIPEGCN_REF"]).resolve()

CONFIGS = {
    "sync_p2": dict(n_parts=2),
    "sync_corr_p2": dict(n_parts=2, feat_corr=True, grad_corr=True, corr_momentum=0.9),
    "pipeline_p2": dict(n_parts=2, enable_pipeline=True),
    "pipeline_corr_p3": dict(n_parts=3, enable_pipeline=True, feat_corr=True, grad_corr=True, corr_momentum=0.95),
    "pipeline_pp_p2": dict(n_parts=2, enable_pipeline=True, use_pp=True),
}
N_EPOCHS, N_LAYERS, N_HIDDEN, N_CLASS, SEED = 3, 3, 16, 5, 0


def worker(rank, size, name, cfg, port, q):
    sys.path.insert(0, str(ROOT))
    import torch
    torch.set_num_threads(1)
    from tests.golden import ref_shims
    ref_shims.install_cuda_shims()
    ref_shims.install_dgl_shim()
    sys.path.insert(0, str(REF))                      # reference modules win over same-named repo files
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=size)

    import dgl                                         # the shim
    import train as T                                  # PipeGCN/train.py  (star-imports helper.utils, module.model)
    from helper import context as ctx                  # PipeGCN/helper/context.py
    assert T.__file__.startswith(str(REF)) and ctx.__file__.startswith(str(REF))
    import torch.nn.functional as F

    from oracle import dglpart
    from pipegcn_b200.synthetic import make_graph, random_partition

    g = make_graph("tiny")
    part = random_partition(g.n_nodes, size)
    parts = dglpart.partition_graph(g.n_nodes, g.src, g.dst, part, size, g.feat, g.label, g.train_mask)
    p = parts[rank]
    graph = ref_shims.FakeGraph(p.su, p.sv, n_u=p.n_nodes)
    node_dict = dict(p.node_dict)
    node_dict[dgl.NID] = node_dict.pop(dglpart.NID)
    gpb = p.gpb
    args = argparse.Namespace(model="graphsage", use_pp=cfg.get("use_pp", False), norm="layer", dropout=0.0, n_linear=0,
                              n_train=int(g.train_mask.sum()), n_feat=g.n_feat, n_hidden=N_HIDDEN, n_class=N_CLASS,
                              n_layers=N_LAYERS, backend="gloo", enable_pipeline=cfg.get("enable_pipeline", False),
                              feat_corr=cfg.get("feat_corr", False), grad_corr=cfg.get("grad_corr", False),
                              corr_momentum=cfg.get("corr_momentum", 0.95), seed=SEED, lr=1e-2, weight_decay=0)

    # ---- PipeGCN/train.py:262-305, the reference's own functions -------------------------------------
    part_g = T.create_inner_graph(graph.clone(), node_dict)
    num_in = node_dict["inner_node"].bool().sum().item()
    graph, part_g, node_dict = T.move_to_cuda(graph, part_g, node_dict)
    boundary = T.get_boundary(node_dict, gpb)
    layer_size = T.get_layer_size(args.n_feat, args.n_hidden, args.n_class, args.n_layers)
    pos = T.get_pos(node_dict, gpb)
    graph = T.order_graph(part_g, graph, gpb, node_dict, pos)
    in_deg = node_dict["in_degree"]
    graph, node_dict, boundary = T.move_train_first(graph, node_dict, boundary)
    recv_shape = T.get_recv_shape(node_dict)
    ctx.buffer.init_buffer(num_in, graph.num_nodes("_U"), boundary, recv_shape, layer_size[:args.n_layers - args.n_linear],
                           use_pp=args.use_pp, backend=args.backend, pipeline=args.enable_pipeline,
                           corr_feat=args.feat_corr, corr_grad=args.grad_corr, corr_momentum=args.corr_momentum)
    if args.use_pp:                                        # train.py:287-288, the reference's own precompute
        node_dict["feat"] = T.precompute(graph, node_dict, boundary, recv_shape, args)
    labels = node_dict["label"][node_dict["train_mask"]]
    train_mask = node_dict["train_mask"]
    torch.manual_seed(args.seed)
    model = T.create_model(layer_size, args)
    model.cuda()
    ctx.reducer.init(model)
    for i, (pname, param) in enumerate(model.named_parameters()):
        param.register_hook(T.reduce_hook(param, pname, args.n_train))
    loss_fcn = torch.nn.CrossEntropyLoss(reduction="sum")
    optimizer = torch.optim.Adam(model.parameters(), lr=args.lr, weight_decay=args.weight_decay)
    feat = node_dict["feat"]

    u, v = graph.edges()
    out = {"layout": dict(num_in=num_in, num_all=graph.num_nodes("_U"), u=u.long().clone(), v=v.long().clone(),
                          boundary=[None if b is None else b.clone() for b in boundary], recv_shape=list(recv_shape),
                          in_deg=in_deg.clone(), feat=feat.clone(), label=node_dict["label"][:num_in].clone(),
                          train_mask=train_mask[:num_in].clone()),
           "init_state": {k: t.clone() for k, t in model.state_dict().items()}, "epochs": []}

    rec = {}

    def hook(i):
        def fn(mod, inp, outp):
            src = inp[1] if len(inp) > 1 else inp[0]
            rec[i] = dict(f_buf=src.detach().clone(), layer_out=outp.detach().clone())
        return fn
    for i, layer in enumerate(model.layers):
        layer.register_forward_hook(hook(i))

    # ---- PipeGCN/train.py:341-362 ------------------------------------------------------------------------
    for epoch in range(N_EPOCHS):
        state = {k: t.clone() for k, t in model.state_dict().items()}
        model.train()
        logits = model(graph, feat, in_deg)
        loss = loss_fcn(logits[train_mask], labels)
        optimizer.zero_grad(set_to_none=True)
        loss.backward()
        ctx.buffer.next_epoch()
        ctx.reducer.synchronize()
        grads = {n: p_.grad.detach().clone() for n, p_ in model.named_parameters()}
        optimizer.step()
        ctx.comm_timer.clear()
        out["epochs"].append(dict(state=state, layers={i: dict(r) for i, r in rec.items()}, logits=logits.detach().clone(),
                                  loss=float(loss.item()), grads=grads))
    # drain the reference's async transfers of the last epoch before the group goes away
    ctx.buffer._pool.close()
    ctx.buffer._pool.join()
    dist.barrier()
    torch.save(out, q + f"/{name}_{rank}.pt")
    dist.destroy_process_group()


def main():
    import torch
    import torch.multiprocessing as mp
    mp.set_start_method("spawn", force=True)
    sys.path.insert(0, str(ROOT))
    from pipegcn_b200.synthetic import make_graph, random_partition
    for k, (name, cfg) in enumerate(CONFIGS.items()):
        size = cfg["n_parts"]
        import tempfile
        tmp = tempfile.mkdtemp(prefix="pg_golden_")
        procs = [mp.Process(target=worker, args=(r, size, name, cfg, 29700 + k, tmp)) for r in range(size)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=600)
            assert p.exitcode == 0, f"reference worker failed ({name})"
        got = {r: torch.load(f"{tmp}/{name}_{r}.pt") for r in range(size)}
        g = make_graph("tiny")
        fixture = {
            "about": "outputs of the unmodified reference (GATECH-EIC/PipeGCN @ 73ab949) run by tests/golden/make_golden.py",
            "config": dict(cfg, n_epochs=N_EPOCHS, n_layers=N_LAYERS, n_hidden=N_HIDDEN, n_class=N_CLASS, seed=SEED,
                           shape="tiny", dropout=0.0, lr=1e-2),
            "graph": dict(n_nodes=g.n_nodes, src=g.src, dst=g.dst, feat=g.feat, label=g.label, train_mask=g.train_mask,
                          part=random_partition(g.n_nodes, size)),
            "ranks": [got[r] for r in range(size)],
        }
        # the reducer must have produced identical gradients on every rank (reducer.py:30)
        for e in range(N_EPOCHS):
            for n, t in got[0]["epochs"][e]["grads"].items():
                for r in range(1, size):
                    assert torch.equal(t, got[r]["epochs"][e]["grads"][n]), (name, e, n)
        path = HERE / f"ref_{name}.pt"
        torch.save(fixture, path)
        print(f"wrote {path} ({path.stat().st_size / 1024:.0f} KiB); losses rank0 "
              f"{[round(ep['loss'], 4) for ep in got[0]['epochs']]}")


if __name__ == "__main__":
    main()
