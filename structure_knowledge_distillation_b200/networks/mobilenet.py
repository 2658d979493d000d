"""MobileNetV2 (Sandler et al., "MobileNetV2: Inverted Residuals and Linear Bottlenecks", CVPR 2018) as a distillation student:
torchvision's `mobilenet_v2()` features[0..17] (width 1.0, without the 320 -> 1280 layer and the classifier), dilated to output stride 8,
with the ResNet18 student's PSP / DSN head -- computed by the sm_90a kernels of libskd_b200.

Output stride 8 follows CSAIL's MobileNetV2dilated rule: features[7..13] dilate 2, features[14..17] dilate 4; a 3x3 convolution with
stride 2 there gets stride 1 and dilation = padding = dilate / 2, any other 3x3 convolution dilation = padding = dilate.  The
depthwise shapes are then (stride, dilation) = (2, 1), (1, 1), (1, 2) and (1, 4).

The modules are parameter containers with torchvision's names for the backbone (`features.4.conv.1.0.weight`,
`features.4.conv.1.1.running_var`, ...) and the ResNet18 student's for the head (`pspmodule.*`, `head.*`, `dsn.*`), so a torchvision
ImageNet state dict initialises the backbone through load_S_model's key intersection.  A depthwise weight is the torch (C, 1, 3, 3)
parameter.  forward returns the 7-list `[x, x_dsn, x_feat_after_psp, f17, f13, f6, f3]`: the PSP feature at index -5 for the
pair-wise loss, the DSN head (on features[13], 96 channels at 1/8) at index 1.

The backbone's convolutions run in split-precision 3xTF32 (`precise`) in the forward pass, the head's in TF32 as the ResNet18
student's layer3 / layer4 / head do (DESIGN.md "MobileNetV2 student" has the measured error of both choices).
"""
import math

import torch
import torch.nn as nn

from .. import functions as Fn
from .. import ops
from ..libs import InPlaceABNSync
from .pspnet_combine import Conv2d, PSPModule, _Dropout2d

# (expansion t, output channels c, repeats n, first stride s) of torchvision's mobilenet_v2, width 1.0
SETTINGS = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1))


def dilate_of(index):
    """CSAIL's MobileNetV2dilated (output stride 8): the dilate factor of features[index]."""
    return 4 if index >= 14 else (2 if index >= 7 else 1)


def dw_geometry(stride, dilate):
    """-> (stride, dilation) of a depthwise 3x3 convolution of torchvision stride `stride` in a block dilated by `dilate`."""
    if dilate == 1:
        return stride, 1
    if stride == 2:
        return 1, dilate // 2
    return 1, dilate


def block_specs():
    """-> [(index, cin, cout, t, torchvision stride)] of features[1..17]."""
    out, cin, i = [], 32, 1
    for t, c, n, s in SETTINGS:
        for k in range(n):
            out.append((i, cin, c, t, s if k == 0 else 1))
            cin, i = c, i + 1
    return out


class DepthwiseConv(nn.Module):
    """nn.Conv2d(C, C, 3, stride, padding=dilation, dilation, groups=C, bias=False) parameter container (weight (C, 1, 3, 3), torch's
    default init)."""

    def __init__(self, channels, stride, dilation):
        super().__init__()
        self.channels, self.stride, self.dilation = channels, stride, dilation
        ops.dwconv_check(channels, (channels, 1, 3, 3), stride, dilation)
        w = torch.empty(channels, 1, 3, 3)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        self.weight = nn.Parameter(w)

    def extra_repr(self):
        return "{channels}, stride={stride}, dilation={dilation}".format(**self.__dict__)


def _bn_act(bn, x, training, relu6, residual=None):
    return Fn.MbBnAct.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked, training, bn.momentum,
                            bn.eps, relu6, residual)


class InvertedResidual(nn.Module):
    """1x1 expand (omitted when t = 1) -> BN -> ReLU6 -> depthwise 3x3 -> BN -> ReLU6 -> 1x1 project -> BN (+ input when stride 1
    and cin = cout); `conv` holds torchvision's layers in torchvision's order."""

    def __init__(self, cin, cout, t, stride, dilate):
        super().__init__()
        hidden = cin * t
        s, d = dw_geometry(stride, dilate)
        self.use_res_connect = stride == 1 and cin == cout
        layers = []
        if t != 1:
            layers.append(nn.Sequential(Conv2d(cin, hidden, 1, bias=False), nn.BatchNorm2d(hidden)))
        layers += [nn.Sequential(DepthwiseConv(hidden, s, d), nn.BatchNorm2d(hidden)), Conv2d(hidden, cout, 1, bias=False),
                   nn.BatchNorm2d(cout)]
        self.conv = nn.Sequential(*layers)

    def forward(self, x, precise=True):
        layers = list(self.conv)
        h = x
        if len(layers) == 4:
            expand = layers.pop(0)
            h = _bn_act(expand[1], Fn.Conv2d.apply(h, expand[0].weight, None, 1, 0, 1, precise), self.training, True)
        dw, project, bn = layers
        h = Fn.MbDwBnRelu6.apply(h, dw[0].weight, dw[1].weight, dw[1].bias, dw[1].running_mean, dw[1].running_var,
                                 dw[1].num_batches_tracked, dw[0].stride, dw[0].dilation, self.training, dw[1].momentum, dw[1].eps)
        h = Fn.Conv2d.apply(h, project.weight, None, 1, 0, 1, precise)
        return _bn_act(bn, h, self.training, False, x if self.use_res_connect else None)


class MobileNetV2Dilated(nn.Module):
    """MobileNetV2 backbone at output stride 8 plus the ResNet18 student's PSP module (320 -> 128), DSN head on features[13] and
    classifier.  H and W: any size (the 1/8 maps are ceil-divided: 64x128 at 512x1024, 45x60 at 360x480)."""

    def __init__(self, classes=19):
        super().__init__()
        feats = [nn.Sequential(Conv2d(3, 32, 3, 2, 1, bias=False), nn.BatchNorm2d(32))]
        feats += [InvertedResidual(cin, cout, t, s, dilate_of(i)) for i, cin, cout, t, s in block_specs()]
        self.features = nn.Sequential(*feats)
        self.pspmodule = PSPModule(320, 128)
        self.head = Conv2d(128, classes, 1, bias=True)
        self.dsn = nn.Sequential(Conv2d(96, 128, 3, 1, 1), InPlaceABNSync(128), _Dropout2d(0.1), Conv2d(128, classes, 1, bias=True))
        self.classes = classes
        self.precise = True

    def dropouts(self):
        return [self.pspmodule.bottleneck[2], self.dsn[2]]

    def level_channels(self):
        """Widths of preds[-1] .. preds[-5]: features[3], [6], [13], [17] (their projection's output) and the PSP features."""
        return tuple(self.features[i].conv[-2].out_channels for i in (3, 6, 13, 17)) + (self.pspmodule.bottleneck[0].out_channels,)

    def forward(self, x):
        # the (N,3,H,W) image, or the 4-channel NHWC image NetModel.forward builds for the teacher
        x = ops.pad_channels(x, 4) if x.shape[1] == 3 else ops.to_nhwc(x)
        precise = self.precise
        stem = self.features[0]
        h = _bn_act(stem[1], Fn.Conv2d.apply(x, stem[0].weight, None, 2, 1, 1, precise), self.training, True)
        keep = {}
        for i in range(1, 18):
            h = self.features[i](h, precise)
            if i in (3, 6, 13, 17):
                keep[i] = h
        f3, f6, f13, f17 = keep[3], keep[6], keep[13], keep[17]
        bn, drop = self.dsn[1], self.dsn[2]
        x_dsn = self.dsn[3](bn(self.dsn[0](f13), chan_mul=drop.channel_multiplier(f13.shape[0], bn.num_features, f13.device)))
        feat = self.pspmodule(f17)
        return [self.head(feat), x_dsn, feat, f17, f13, f6, f3]


def MobileNetV2(classes=19):
    return MobileNetV2Dilated(classes)
