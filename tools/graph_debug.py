"""Bisect which part of an epoch invalidates CUDA-graph capture."""
import os, sys, traceback
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch
from oracle.train import initial_state
from pipegcn_b200 import ops
from pipegcn_b200.train import RankEngine
from pipegcn_b200.world import LocalWorld
from tests.helpers import make_args, small_world

g, _, layouts, setups = small_world("tiny", 1)
mode = os.environ.get("CAPMODE", "global")
for what in ("forward", "fwd_bwd", "fwd_bwd_next", "fwd_bwd_reduce", "full"):
    oargs, eargs = make_args(g, 5, n_epochs=4, enable_pipeline=True)
    eargs.cuda_graph = True
    eargs.dtype = os.environ.get("DT", "fp32")
    eng = RankEngine(layouts[0], eargs, LocalWorld(1, "cuda").view(0), init_state=initial_state(oargs), seg_len=32)
    for _ in range(3):
        eng.run_epoch()
    eng.buffer.graph_mode = True
    ops.STEP_DEV = eng.buffer.epoch_dev
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    eng.optimizer.zero_grad(set_to_none=True)
    try:
        with torch.cuda.graph(gr, capture_error_mode=mode):
            if what == "forward":
                eng.model.train()
                logits = eng.model(eng.graph, eng.buffer.inner_view(0), eng.in_deg)
            else:
                loss = eng.forward_backward()
                if what == "fwd_bwd_next":
                    eng.buffer.next_epoch()
                elif what == "fwd_bwd_reduce":
                    eng.buffer.next_epoch(); eng.reducer.synchronize()
                elif what == "full":
                    eng.finish_epoch()
        gr.replay(); torch.cuda.synchronize()
        print(f"[graph_debug] mode={mode} {what}: OK", flush=True)
    except Exception as e:
        print(f"[graph_debug] mode={mode} {what}: FAIL {type(e).__name__} {str(e)[:150]}", flush=True)
        torch.cuda.synchronize()
    ops.STEP_DEV = None
    del eng, gr
