"""InPlace-ABN module facade with the reference's constructor surface (libs/bn.py:48-193), backed by the fused NHWC
sm_90a kernels (csrc/abn.cu).  State-dict names are the reference's: weight, bias, running_mean, running_var.

`InPlaceABNSync` keeps its name and arguments; with one process per GPU the statistics are per-rank by default (what
the reference's own launch script runs: 1 GPU, run_train_val.sh:8-15).
"""
import torch
import torch.nn as nn

from .. import functions as Fn

ACT_LEAKY_RELU, ACT_ELU, ACT_NONE = "leaky_relu", "elu", "none"


class InPlaceABN(nn.Module):
    """InPlace Activated Batch Normalization"""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, activation="leaky_relu", slope=0.01):
        super().__init__()
        self.num_features, self.affine, self.eps, self.momentum = num_features, affine, eps, momentum
        self.activation, self.slope = activation, slope
        if affine:
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
        else:
            self.register_parameter('weight', None)
            self.register_parameter('bias', None)
        self.register_buffer('running_mean', torch.zeros(num_features))
        self.register_buffer('running_var', torch.ones(num_features))

    def reset_parameters(self):
        self.running_mean.zero_(); self.running_var.fill_(1)
        if self.affine:
            self.weight.data.fill_(1); self.bias.data.zero_()

    def forward(self, x, residual=None, fuse_relu=False, chan_mul=None):
        """residual / fuse_relu / chan_mul fold the ops that follow this layer in the PSPNet graph into the same pass:
        `relu(abn(x) + residual)` (pspnet_combine.py:42-43,81-82) and `Dropout2d(abn(x))` (:99,143)."""
        act = self.activation
        if fuse_relu:
            if act != ACT_NONE:
                raise ValueError("fuse_relu needs activation='none'")
            act = "relu"
        elif residual is not None:
            raise ValueError("a fused residual add is only defined together with fuse_relu")
        return Fn.ABN.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.training, self.momentum,
                            self.eps, act, self.slope, residual, chan_mul, getattr(self, "sync_stats", False))

    def __repr__(self):
        rep = '{name}({num_features}, eps={eps}, momentum={momentum}, affine={affine}, activation={activation}'
        rep += ' slope={slope})' if self.activation == "leaky_relu" else ')'
        return rep.format(name=self.__class__.__name__, **self.__dict__)


class InPlaceABNSync(InPlaceABN):
    """Same constructor as libs/bn.py:108-147 (`devices` accepted and ignored: one process per GPU).  `sync_stats = True` (per module,
    or NetModel's `args.sync_bn`) synchronises the batch statistics across the ranks of the default process group the way the
    reference's multi-GPU mode does across its worker threads (libs/functions.py:177-209,255-283); the default keeps them per rank,
    which is what the reference's own launch script runs (one GPU)."""
    sync_stats = False

    def __init__(self, num_features, devices=None, eps=1e-5, momentum=0.1, affine=True, activation="leaky_relu", slope=0.01):
        super().__init__(num_features, eps, momentum, affine, activation, slope)
        self.devices = devices


class ABN(nn.Sequential):
    """Activated Batch Normalization (libs/bn.py:24-45)."""

    def __init__(self, num_features, activation=nn.ReLU(inplace=True), **kwargs):
        from collections import OrderedDict
        super().__init__(OrderedDict([("bn", nn.BatchNorm2d(num_features, **kwargs)), ("act", activation)]))


class InPlaceABNWrapper(nn.Module):
    def __init__(self, *args, **kwargs):
        super().__init__()
        self.bn = InPlaceABN(*args, **kwargs)

    def forward(self, input):
        return self.bn(input)


class InPlaceABNSyncWrapper(nn.Module):
    def __init__(self, *args, **kwargs):
        super().__init__()
        self.bn = InPlaceABNSync(*args, **kwargs)

    def forward(self, input):
        return self.bn(input)
