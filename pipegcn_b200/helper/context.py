"""Process-global hot-path objects -- the plug-in seam of the reference.

PipeGCN/helper/context.py:4-5 holds `buffer = Buffer()` and
`reducer = Reducer()`; model code reaches them as `ctx.buffer` / `ctx.reducer`
(PipeGCN/module/model.py:46, PipeGCN/train.py:283,302,357,360).
Replacing these two objects is how this engine drops in.
"""
from .feature_buffer import Buffer
from .reducer import Reducer
from .timer.timer import comm_timer

buffer = Buffer()
reducer = Reducer()
