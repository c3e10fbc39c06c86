"""`Reducer`: gradient all-reduce, kept as a plain NCCL call (BASELINE north_star).

Semantics of PipeGCN/helper/reducer.py:23-33 + train.py:200-203,304-305:
every parameter gradient becomes  sum over ranks of (grad / n_train)  with n_train the
GLOBAL number of training nodes.  The reference copies each gradient to pinned host
memory and all-reduces it over gloo in its own process group from a pool thread; here
all gradients are packed into one flat fp32 bucket, scaled, reduced with a single
`ncclAllReduce` on the compute stream and unpacked -- stream-ordered, no host sync.
"""
import torch


class Reducer(object):

    def __init__(self, world=None):
        super().__init__()
        self._world = world
        self._params = []
        self._pending = {}
        self._n_train = None
        self.flat = None

    def init(self, model, world=None):
        if world is not None:
            self._world = world
        if self._world is None:
            from ..world import default_world
            self._world = default_world()
        self._params = [(n, p) for n, p in model.named_parameters()]
        total = sum(p.numel() for _, p in self._params)
        dev = self._params[0][1].device if self._params else 'cpu'
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self._pending = {}

    def reduce(self, param, name, data, n_train):
        """Called from the parameter hook with the local gradient (train.py:200-203)."""
        self._pending[name] = data
        self._n_train = n_train

    def synchronize(self):
        """Pack, scale by 1/n_train, all-reduce (SUM), write back into `param.grad`."""
        if not self._params:
            return
        self.pack()
        if self._world.size > 1:
            self._world.all_reduce_sum_(self.flat)
        self.unpack()

    def pack(self):
        """flat <- concat(grad) / n_train.  (`synchronize` = pack, all-reduce, unpack.)"""
        grads = []
        for name, p in self._params:
            g = self._pending.get(name, p.grad)
            if g is None:
                g = torch.zeros_like(p)
            grads.append(g)
        views, off = [], 0
        for g in grads:
            views.append(self.flat[off: off + g.numel()].view_as(g))
            off += g.numel()
        torch._foreach_copy_(views, grads)
        if self._n_train is not None:
            self.flat.div_(self._n_train)
        self._views = views

    def unpack(self):
        for (name, p), v in zip(self._params, self._views):
            if p.grad is None:
                p.grad = v.clone()
            else:
                p.grad.copy_(v)
        self._pending.clear()
