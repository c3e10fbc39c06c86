"""`CommTimer`: exposed (non-overlapped) communication time per epoch.

Keeps the interface of PipeGCN/helper/timer/comm_timer.py:6-33 -- named
sections `forward_<l>` / `backward_<l>`, `tot_time()`, `clear()`, duplicate names
raise -- but measures on the device: a section is the pair of CUDA events that
brackets the flag-wait kernel on the compute stream, i.e. the time the compute
stream was blocked on the exchange (the reference times the host blocking in
`r.wait()` / event waits, feature_buffer.py:146,155,223,230).
"""
import time
from contextlib import contextmanager


class CommTimer(object):

    def __init__(self):
        super().__init__()
        self._time = {}
        self._events = {}

    def _claim(self, name):
        if name in self._time or name in self._events:
            raise Exception(name + " already exists")

    @contextmanager
    def timer(self, name):
        """Host wall-clock section (reference-compatible)."""
        self._claim(name)
        t0 = time.time()
        yield
        self._time[name] = (t0, time.time())

    def add_events(self, name, start, end):
        """Device section: two recorded torch.cuda.Event(enable_timing=True)."""
        self._claim(name)
        self._events[name] = (start, end)

    def tot_time(self):
        """Seconds; synchronises on the recorded events."""
        tot = 0.0
        for (t0, t1) in self._time.values():
            tot += t1 - t0
        for (e0, e1) in self._events.values():
            e1.synchronize()
            tot += e0.elapsed_time(e1) * 1e-3
        return tot

    def sections(self):
        out = {k: t1 - t0 for k, (t0, t1) in self._time.items()}
        for k, (e0, e1) in self._events.items():
            e1.synchronize()
            out[k] = e0.elapsed_time(e1) * 1e-3
        return out

    def print_time(self):
        import torch.distributed as dist
        rank = dist.get_rank() if dist.is_initialized() else 0
        for k, v in self.sections().items():
            print(f'(rank {rank}) Communication time of {k}: {v} seconds.')

    def clear(self):
        self._time = {}
        self._events = {}
