"""`SyncBatchNorm` for `--norm batch` (PipeGCN/module/sync_bn.py:7-56).

Batch statistics over the rows of ALL partitions: sum(x) and sum(x^2) are all-reduced in the forward, sum(g) and
sum(g * x_hat) in the backward; `whole_size` is the divisor (the reference passes the global number of training
nodes, train.py:194-195).  Four [d]-sized all-reduces per layer -- plain NCCL calls, no custom kernel (SURVEY.md
§2.1 #4 keeps it out of the hot path).  state_dict keys as the reference: weight, bias, running_mean, running_var.
"""
import torch
import torch.distributed as dist
from torch import nn
from torch.autograd import Function


def _all_reduce(t):
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


class _SyncBN(Function):

    @staticmethod
    def forward(ctx, x, weight, bias, whole_size, running_mean, running_var, training, momentum, eps):
        xf = x.float()
        if training:
            stats = torch.stack([xf.sum(0), (xf * xf).sum(0)])
            _all_reduce(stats)
            mean = stats[0] / whole_size
            var = (stats[1] - mean * stats[0]) / whole_size
            running_mean.mul_(1 - momentum).add_(mean * momentum)
            running_var.mul_(1 - momentum).add_(var * momentum)
        else:
            mean, var = running_mean, running_var
        std = torch.sqrt(var + eps)
        x_hat = (xf - mean) / std
        if training:
            ctx.save_for_backward(x_hat, weight, std)
            ctx.whole_size = whole_size
        return (x_hat * weight + bias).to(x.dtype)

    @staticmethod
    def backward(ctx, grad):
        x_hat, weight, std = ctx.saved_tensors
        g = grad.float()
        red = torch.stack([g.sum(0), (g * x_hat).sum(0)])
        _all_reduce(red)
        dbias, dweight = red[0], red[1]
        n = ctx.whole_size
        dx = (weight / n) / std * (n * g - dbias - x_hat * dweight)
        return dx.to(grad.dtype), dweight, dbias, None, None, None, None, None, None


class SyncBatchNorm(nn.Module):

    def __init__(self, num_features, whole_size, eps=1e-5, momentum=0.1):
        super().__init__()
        self.register_buffer('running_mean', torch.zeros(num_features))
        self.register_buffer('running_var', torch.ones(num_features))
        self.whole_size, self.eps, self.momentum = whole_size, eps, momentum
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))

    def forward(self, x):
        return _SyncBN.apply(x, self.weight, self.bias, self.whole_size, self.running_mean, self.running_var,
                             self.training, self.momentum, self.eps)
