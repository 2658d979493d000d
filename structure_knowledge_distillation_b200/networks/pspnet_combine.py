"""PSPNet / dilated ResNet with the reference's public surface (networks/pspnet_combine.py): `Res_pspnet(block, layers,
num_classes)`, `BasicBlock`, `Bottleneck`, `PSPModule`, identical state-dict names and the 7-tensor output list
`[x, x_dsn, x_feat_after_psp, x4, x3, x2, x1]` (:189) -- computed by the sm_90a kernels of libskd_b200.

Two execution paths over the same parameters:
  * training (student): torch.autograd.Functions, conv (wgmma) -> fused ABN(+ReLU / +residual+ReLU / +Dropout2d);
  * frozen  (teacher: eval() under no_grad, networks/kd_model.py:121-122): no autograd, eval-mode ABN folded into the
    convolution epilogue (scale/shift/activation/residual in registers), layer4 writes straight into the PSP concat
    buffer -- one kernel per conv, nothing else touches HBM.
Activations are NHWC in memory and (N,C,H,W) in shape, so the returned tensors index like the reference's.
"""
import functools
import math

import torch
import torch.nn as nn

from .. import functions as Fn
from .. import ops
from ..libs import InPlaceABN, InPlaceABNSync

affine_par = True
BatchNorm2d = functools.partial(InPlaceABNSync, activation='none')          # pspnet_combine.py:12


class Conv2d(nn.Module):
    """nn.Conv2d stand-in (same constructor arguments, parameter names and default init) whose weight lives in OHWI
    (channels-last) storage, the K-major layout the wgmma kernels read."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, bias=True):
        super().__init__()
        k = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
        self.in_channels, self.out_channels, self.kernel_size = in_channels, out_channels, (k, k)
        self.stride, self.padding, self.dilation = stride, padding, dilation
        self.precise = False              # training forward in split-precision 3xTF32 (set for the student's stem, layer1 and layer2)
        w = torch.empty(out_channels, in_channels, k, k)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))                         # nn.Conv2d.reset_parameters
        self.weight = nn.Parameter(w.contiguous(memory_format=torch.channels_last))
        if bias:
            bound = 1 / math.sqrt(in_channels * k * k)
            self.bias = nn.Parameter(torch.empty(out_channels).uniform_(-bound, bound))
        else:
            self.register_parameter('bias', None)

    def forward(self, x):
        return Fn.Conv2d.apply(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.precise)

    def frozen(self, x, scale=None, shift=None, residual=None, act="none", slope=0.0, out=None):
        if Fn._small_cin(self.weight) and self.bias is None and residual is None and out is None:
            y, _ = Fn.conv_forward_small_cin(x, self.weight, self.stride, self.padding, self.dilation, scale=scale, shift=shift,
                                             act=act, slope=slope)
            return y
        y, _ = Fn.conv_forward_padded(x, self.weight, self.bias, self.stride, self.padding, self.dilation, scale=scale,
                                      shift=shift, residual=residual, act=act, slope=slope, out=out)
        return y

    def extra_repr(self):
        return '{in_channels}, {out_channels}, kernel_size={kernel_size}, stride={stride}, padding={padding}, dilation={dilation}'.format(**self.__dict__)


def conv3x3(in_planes, out_planes, stride=1):
    "3x3 convolution with padding"
    return Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


def _fold(bn):
    """eval-mode ABN -> per-channel (scale, shift) for a conv epilogue (libs/src/bn.cu:140-165 with running stats).
    Cached only for FROZEN modules (the teacher: requires_grad False), where a checkpoint load (copy_ bumps the version counters)
    is the only thing that can change the inputs.  Trainable modules are folded afresh on every eval forward: their statistics
    and affine parameters are written through raw pointers by the stats / SGD kernels, which no version counter sees."""
    if bn.weight is not None and bn.weight.requires_grad:
        return ops.abn_fold(bn.running_mean, bn.running_var, bn.weight, bn.bias, bn.eps)
    key = (bn.weight._version, bn.bias._version, bn.running_mean._version, bn.running_var._version,
           bn.weight.data_ptr(), bn.running_mean.data_ptr())
    cached = getattr(bn, "_folded", None)
    if cached is None or cached[0] != key:
        cached = (key, ops.abn_fold(bn.running_mean, bn.running_var, bn.weight, bn.bias, bn.eps))
        bn._folded = cached
    return cached[1]


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, multi_grid=1):
        super().__init__()
        dilation = dilation * multi_grid
        self.conv1 = Conv2d(inplanes, planes, 3, stride, dilation, dilation, bias=False)
        self.bn1 = BatchNorm2d(planes)
        self.conv2 = Conv2d(planes, planes, 3, 1, dilation, dilation, bias=False)
        self.bn2 = BatchNorm2d(planes)
        self.downsample = downsample

    def forward(self, x):
        residual = x if self.downsample is None else self.downsample[1](self.downsample[0](x))
        out = self.bn1(self.conv1(x), fuse_relu=True)
        return self.bn2(self.conv2(out), residual=residual, fuse_relu=True)

    def frozen(self, x, out=None):
        residual = x if self.downsample is None else self.downsample[0].frozen(x, *_fold(self.downsample[1]))
        o = self.conv1.frozen(x, *_fold(self.bn1), act="relu")
        return self.conv2.frozen(o, *_fold(self.bn2), residual=residual, act="relu", out=out)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, fist_dilation=1, multi_grid=1):
        super().__init__()
        self.conv1 = Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = BatchNorm2d(planes)
        self.conv2 = Conv2d(planes, planes, 3, stride, dilation * multi_grid, dilation * multi_grid, bias=False)
        self.bn2 = BatchNorm2d(planes)
        self.conv3 = Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.dilation, self.stride = dilation, stride

    def forward(self, x):
        residual = x if self.downsample is None else self.downsample[1](self.downsample[0](x))
        out = self.bn1(self.conv1(x), fuse_relu=True)
        out = self.bn2(self.conv2(out), fuse_relu=True)
        return self.bn3(self.conv3(out), residual=residual, fuse_relu=True)

    def frozen(self, x, out=None, o1=None, chain=None):
        """o1: this block's conv1 output, already computed by the previous block's chained launch.  chain: the next block, whose
        conv1 then runs in the same launch as this block's conv3 (ops.conv1x1_chain) -> (output, the next block's conv1 output)."""
        residual = x if self.downsample is None else self.downsample[0].frozen(x, *_fold(self.downsample[1]))
        o = o1 if o1 is not None else self.conv1.frozen(x, *_fold(self.bn1), act="relu")
        o = self.conv2.frozen(o, *_fold(self.bn2), act="relu")
        if chain is not None:
            return ops.conv1x1_chain(o, ops.weight_ohwi(self.conv3.weight), *_fold(self.bn3), residual,
                                     ops.weight_ohwi(chain.conv1.weight), *_fold(chain.bn1))
        return self.conv3.frozen(o, *_fold(self.bn3), residual=residual, act="relu", out=out)

    def chains_into(self, nxt):
        """Whether this block's conv3 and `nxt`'s conv1 can run as one launch: 1x1 pair with no downsample between them and a conv1
        output the chained kernel's accumulators hold (layer4's 512 channels do not fit)."""
        return (isinstance(nxt, Bottleneck) and nxt.downsample is None and nxt.conv1.out_channels in ops.CHAIN_COUT1 and
                self.conv3.out_channels % 64 == 0 and self.conv3.in_channels % 4 == 0)


class _Dropout2d(nn.Dropout2d):
    """Dropout2d whose mask multiplication is fused into the preceding ABN pass.  `injected` (N,C) keep-mask for tests."""
    injected = None

    def channel_multiplier(self, n, c, device):
        if not self.training or self.p == 0:
            return None
        if self.injected is not None and (self.injected.device != device or self.injected.dtype != torch.float32):
            self.injected = self.injected.to(device=device, dtype=torch.float32)     # once: a CUDA-graph capture cannot copy from the host
        keep = self.injected if self.injected is not None else (torch.rand(n, c, device=device) >= self.p).float()
        return (keep / (1.0 - self.p)).contiguous()


class PSPModule(nn.Module):
    """Zhao et al., Pyramid scene parsing network (pspnet_combine.py:86-112)."""

    def __init__(self, features, out_features=512, sizes=(1, 2, 3, 6)):
        super().__init__()
        self.sizes = tuple(sizes)
        self.stages = nn.ModuleList([nn.Sequential(nn.AdaptiveAvgPool2d(output_size=(s, s)),
                                                   Conv2d(features, out_features, 1, bias=False),
                                                   InPlaceABNSync(out_features)) for s in sizes])
        self.bottleneck = nn.Sequential(Conv2d(features + len(sizes) * out_features, out_features, 3, padding=1, dilation=1, bias=False),
                                        InPlaceABNSync(out_features), _Dropout2d(0.1))

    def _stage_inputs(self, pooled):
        off = 0
        for s in self.sizes:                               # (N, s*s, C) -> NHWC-stored (N, C, s, s)
            yield s, pooled[:, off:off + s * s].contiguous().view(pooled.shape[0], s, s, pooled.shape[2]).permute(0, 3, 1, 2)
            off += s * s

    def forward(self, feats):
        n, c, h, w = feats.shape
        pooled = Fn.PspPool.apply(feats, self.sizes)
        outs = []
        for (s, xin), stage in zip(self._stage_inputs(pooled), self.stages):
            y = stage[2](stage[1](xin))
            outs.append(y.permute(0, 2, 3, 1).reshape(n, s * s, -1))
        cat = Fn.PspAssemble.apply(feats, self.sizes, *outs)
        bn, drop = self.bottleneck[1], self.bottleneck[2]
        return bn(self.bottleneck[0](cat), chan_mul=drop.channel_multiplier(n, bn.num_features, feats.device))

    def frozen(self, cat, feats_view):
        """`cat` is the concat buffer whose last channels already hold layer4's output (`feats_view`)."""
        n = cat.shape[0]
        pooled = ops.psp_pool_fwd(feats_view, list(self.sizes))
        cs = self.stages[0][1].out_channels
        for i, ((s, xin), stage) in enumerate(zip(self._stage_inputs(pooled), self.stages)):
            y = stage[1].frozen(xin, *_fold(stage[2]), act=stage[2].activation, slope=stage[2].slope)
            ops.psp_upsample_fwd(y.permute(0, 2, 3, 1).reshape(n, s * s, cs), s, cat, i * cs)
        bn = self.bottleneck[1]
        return self.bottleneck[0].frozen(cat, *_fold(bn), act=bn.activation, slope=bn.slope)


class ResNet(nn.Module):
    def __init__(self, block, layers, num_classes):
        self.inplanes = 128
        super().__init__()
        self.conv1 = conv3x3(3, 64, stride=2); self.bn1 = BatchNorm2d(64)
        self.conv2 = conv3x3(64, 64); self.bn2 = BatchNorm2d(64)
        self.conv3 = conv3x3(64, 128); self.bn3 = BatchNorm2d(128)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=1, dilation=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=1, dilation=4, multi_grid=(1, 1, 1))
        if list(layers) == [3, 4, 23, 3]:
            c4, cp, c3 = 2048, 512, 1024
        elif list(layers) == [2, 2, 2, 2]:
            c4, cp, c3 = 512, 128, 256
        else:
            raise ValueError('layers should be [3, 4, 23, 3] or [2, 2, 2, 2]')
        self.pspmodule = PSPModule(c4, cp)
        self.head = Conv2d(cp, num_classes, 1, bias=True)
        self.dsn = nn.Sequential(Conv2d(c3, cp, 3, 1, 1), InPlaceABNSync(cp), _Dropout2d(0.1), Conv2d(cp, num_classes, 1, bias=True))
        self.set_precise_early_layers(True)

    def set_precise_early_layers(self, on=True):
        """Training-mode forward of the stem, layer1 and layer2 in split-precision 3xTF32 (fp32-grade): with batch statistics the
        operand rounding of these first layers is what the rest of the network amplifies (DESIGN.md "TF32 and parity").  No effect
        on the frozen / eval path."""
        early = [c for layer in (self.layer1, self.layer2) for c in layer.modules() if isinstance(c, Conv2d)]
        for m in [self.conv1, self.conv2, self.conv3] + early:
            m.precise = bool(on)

    def _make_layer(self, block, planes, blocks, stride=1, dilation=1, multi_grid=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(Conv2d(self.inplanes, planes * block.expansion, 1, stride, bias=False),
                                       BatchNorm2d(planes * block.expansion, affine=affine_par))
        grid = lambda i: multi_grid[i % len(multi_grid)] if isinstance(multi_grid, tuple) else 1
        layers = [block(self.inplanes, planes, stride, dilation=dilation, downsample=downsample, multi_grid=grid(0))]
        self.inplanes = planes * block.expansion
        layers += [block(self.inplanes, planes, dilation=dilation, multi_grid=grid(i)) for i in range(1, blocks)]
        return nn.Sequential(*layers)

    def dropouts(self):
        return [self.pspmodule.bottleneck[2], self.dsn[2]]

    def forward(self, x):
        # the 3-channel image travels as 4 channels (16-byte pixel rows for TMA); a caller that feeds two networks
        # (NetModel.forward) pads once and passes the 4-channel tensor to both
        x = ops.pad_channels(x, 4) if x.shape[1] == 3 else ops.to_nhwc(x)
        if not self.training and not torch.is_grad_enabled():
            return self._forward_frozen(x)
        x = self.bn1(self.conv1(x), fuse_relu=True)
        x = self.bn2(self.conv2(x), fuse_relu=True)
        x = self.bn3(self.conv3(x), fuse_relu=True)
        x = Fn.MaxPool3x3s2.apply(x)
        x1 = self.layer1(x); x2 = self.layer2(x1); x3 = self.layer3(x2)
        n = x3.shape[0]
        bn, drop = self.dsn[1], self.dsn[2]
        x_dsn = self.dsn[3](bn(self.dsn[0](x3), chan_mul=drop.channel_multiplier(n, bn.num_features, x.device)))
        x4 = self.layer4(x3)
        x_feat_after_psp = self.pspmodule(x4)
        x = self.head(x_feat_after_psp)
        return [x, x_dsn, x_feat_after_psp, x4, x3, x2, x1]

    def _forward_frozen(self, x):
        x = self.conv1.frozen(x, *_fold(self.bn1), act="relu")
        x = self.conv2.frozen(x, *_fold(self.bn2), act="relu")
        x = self.conv3.frozen(x, *_fold(self.bn3), act="relu")
        x, _ = ops.maxpool_fwd(x)
        feats = []
        chain = ops.conv1x1_chain_enabled()
        for layer in (self.layer1, self.layer2, self.layer3):
            blocks, o1 = list(layer), None
            for i, blk in enumerate(blocks):
                nxt = blocks[i + 1] if i + 1 < len(blocks) else None
                if chain and isinstance(blk, Bottleneck) and blk.chains_into(nxt):
                    x, o1 = blk.frozen(x, o1=o1, chain=nxt)
                else:
                    x, o1 = (blk.frozen(x, o1=o1) if o1 is not None else blk.frozen(x)), None
            feats.append(x)
        x1, x2, x3 = feats
        bn = self.dsn[1]
        x_dsn = self.dsn[3].frozen(self.dsn[0].frozen(x3, *_fold(bn), act=bn.activation, slope=bn.slope))
        n, _, h, w = x3.shape
        blocks = list(self.layer4)
        c4 = blocks[-1].bn3.num_features if hasattr(blocks[-1], "bn3") else blocks[-1].bn2.num_features
        npri = len(self.pspmodule.sizes) * self.pspmodule.stages[0][1].out_channels
        cat = ops.empty_nhwc(n, npri + c4, h, w, x.device)
        x4 = cat[:, npri:]                                   # layer4's last conv writes its slice of the concat buffer
        y = x3
        for blk in blocks[:-1]:
            y = blk.frozen(y)
        blocks[-1].frozen(y, out=x4)
        x_feat_after_psp = self.pspmodule.frozen(cat, x4)
        x = self.head.frozen(x_feat_after_psp)
        return [x, x_dsn, x_feat_after_psp, x4, x3, x2, x1]


def Res_pspnet(block=Bottleneck, layers=[3, 4, 23, 3], num_classes=21):
    '''
    ResNet(Bottleneck, [3, 4, 23, 3], num_classes)
    ResNet(BasicBlock, [2, 2, 2, 2], num_classes)
    '''
    return ResNet(block, layers, num_classes)
