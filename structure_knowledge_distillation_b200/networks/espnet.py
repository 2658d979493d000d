"""ESPNet-C (Mehta et al., "ESPNet: Efficient Spatial Pyramid of Dilated Convolutions for Semantic Segmentation", ECCV 2018), the
encoder-only ESPNet, and the full ESPNet (ESPNet-C plus its decoder, logits at the input resolution) as distillation students --
computed by the sm_90a kernels of libskd_b200.

The modules are parameter containers (attribute names = state-dict keys: `level1.conv.weight`, `level2_0.d16.conv.weight`,
`level2.0.bn.bn.running_var`, `b2.act.weight`, `classifier.conv.weight`, ...); the computation is the autograd Functions
`EspBnPrelu`, `EspBlock` and `EspConv` of functions.py.  `ESPNet_Encoder.forward` returns the 7-list NetModel and the criteria index:
`[logits, None, feat, level3 out, b2 out, level2 out, b1 out]`, with `feat` (the b3 output, 256 channels at 1/8 resolution) at
index -5 for the pair-wise loss and no auxiliary head at index 1.

Every convolution runs in split-precision 3xTF32 (`precise`), in training and evaluation: train-mode BatchNorm amplifies TF32
operand rounding (DESIGN.md "TF32 and parity"), and the whole network is ~0.6 % of the teacher's forward arithmetic.
"""
import torch
import torch.nn as nn

from .. import functions as Fn
from .. import ops
from .pspnet_combine import Conv2d


def _bnprelu_params(bn, act):
    return (bn.weight, bn.bias, act.weight, bn.running_mean, bn.running_var, bn.num_batches_tracked)


class CBR(nn.Module):
    """Conv k x k / stride s, pad (k-1)/2, no bias -> BatchNorm2d(eps=1e-3) -> PReLU."""

    def __init__(self, nIn, nOut, kSize, stride=1):
        super().__init__()
        self.conv = Conv2d(nIn, nOut, kSize, stride, (kSize - 1) // 2, bias=False)
        self.bn = nn.BatchNorm2d(nOut, eps=1e-3)
        self.act = nn.PReLU(nOut)


class BR(nn.Module):
    """BatchNorm2d(eps=1e-3) -> PReLU."""

    def __init__(self, nOut):
        super().__init__()
        self.bn = nn.BatchNorm2d(nOut, eps=1e-3)
        self.act = nn.PReLU(nOut)


class C(nn.Module):
    def __init__(self, nIn, nOut, kSize, stride=1):
        super().__init__()
        self.conv = Conv2d(nIn, nOut, kSize, stride, (kSize - 1) // 2, bias=False)


class CDilated(nn.Module):
    def __init__(self, nIn, nOut, kSize, stride=1, d=1):
        super().__init__()
        self.conv = Conv2d(nIn, nOut, kSize, stride, (kSize - 1) // 2 * d, dilation=d, bias=False)


class _Esp(nn.Module):
    def _branches(self, nIn, nOut, reduce_k, reduce_s):
        n = nOut // 5
        n1 = nOut - 4 * n
        self.c1 = C(nIn, n, reduce_k, reduce_s)
        self.d1 = CDilated(n, n1, 3, 1, 1)
        self.d2 = CDilated(n, n, 3, 1, 2)
        self.d4 = CDilated(n, n, 3, 1, 4)
        self.d8 = CDilated(n, n, 3, 1, 8)
        self.d16 = CDilated(n, n, 3, 1, 16)

    def _run(self, x, bn, act, stride, add, precise):
        return Fn.EspBlock.apply(x, self.c1.conv.weight, self.d1.conv.weight, self.d2.conv.weight, self.d4.conv.weight,
                                 self.d8.conv.weight, self.d16.conv.weight, bn.weight, bn.bias, act.weight, bn.running_mean,
                                 bn.running_var, bn.num_batches_tracked, stride, add, self.training, bn.momentum, bn.eps, precise)


class DownSamplerB(_Esp):
    """ESP module with a 3x3 / stride-2 reduction; BatchNorm + PReLU held directly on the block (`bn`, `act`)."""

    def __init__(self, nIn, nOut):
        super().__init__()
        self._branches(nIn, nOut, 3, 2)
        self.bn = nn.BatchNorm2d(nOut, eps=1e-3)
        self.act = nn.PReLU(nOut)

    def forward(self, x, precise=True):
        return self._run(x, self.bn, self.act, 2, False, precise)


class DilatedParllelResidualBlockB(_Esp):
    """ESP module with a 1x1 reduction and (add=True) the block input added to the combine; `bn` is a BR."""

    def __init__(self, nIn, nOut, add=True):
        super().__init__()
        self._branches(nIn, nOut, 1, 1)
        self.bn = BR(nOut)
        self.add = add
        if add and nIn != nOut:
            raise ValueError("the residual ESP block needs nIn == nOut")

    def forward(self, x, precise=True):
        return self._run(x, self.bn.bn, self.bn.act, 1, self.add, precise)


class InputProjectionA(nn.Module):
    """`samplingTimes` x AvgPool2d(3, stride 2, padding 1) of the image; no parameters (computed inside the next BR's concat)."""

    def __init__(self, samplingTimes):
        super().__init__()
        self.samplingTimes = samplingTimes


class ESPNet_Encoder(nn.Module):
    """ESPNet-C: `classes` output channels at 1/8 of the input resolution; p residual ESP blocks at level 2, q at level 3."""

    def __init__(self, classes=19, p=2, q=8):
        super().__init__()
        if int(p) < 1 or int(q) < 1:
            raise ValueError("ESPNet-C needs p >= 1 and q >= 1 (got p=%r, q=%r)" % (p, q))
        self.level1 = CBR(3, 16, 3, 2)
        self.sample1 = InputProjectionA(1)
        self.sample2 = InputProjectionA(2)
        self.b1 = BR(16 + 3)
        self.level2_0 = DownSamplerB(16 + 3, 64)
        self.level2 = nn.ModuleList([DilatedParllelResidualBlockB(64, 64) for _ in range(int(p))])
        self.b2 = BR(128 + 3)
        self.level3_0 = DownSamplerB(128 + 3, 128)
        self.level3 = nn.ModuleList([DilatedParllelResidualBlockB(128, 128) for _ in range(int(q))])
        self.b3 = BR(256)
        self.classifier = C(256, classes, 1, 1)
        self.classes = classes
        self.precise = True

    def dropouts(self):
        return []

    def level_channels(self):
        """Widths of preds[-1] .. preds[-5]: b1, level2's output, b2, level3's output and b3 (`feat`)."""
        return (self.b1.bn.num_features, self.level2[-1].bn.bn.num_features, self.b2.bn.num_features,
                self.level3[-1].bn.bn.num_features, self.b3.bn.num_features)

    def _br(self, br, pieces, image=None, ipa=0):
        bn = br.bn
        return Fn.EspBnPrelu.apply(image, ipa, bn.weight, bn.bias, br.act.weight, bn.running_mean, bn.running_var,
                                   bn.num_batches_tracked, self.training, bn.momentum, bn.eps, *pieces)

    def forward(self, x):
        logits, feat, out2, b2, out1, b1 = self._features(x)
        c = self.classes
        return [logits[:, :c], None, feat, out2, b2[:, :131], out1, b1[:, :19]]

    def _features(self, x):
        """-> the channel-padded (logits, feat, out2, b2, out1, b1) (b2: 132 channels, b1: 20; pad channels zero)."""
        # the (N,3,H,W) image, or the 4-channel NHWC image NetModel.forward builds for the teacher
        x = ops.pad_channels(x, 4) if x.shape[1] == 3 else ops.to_nhwc(x)
        precise = self.precise
        c0 = Fn.Conv2d.apply(x, self.level1.conv.weight, None, 2, 1, 1, precise)
        out0, _ = self._br(self.level1, [c0])
        b1, proj1 = self._br(self.b1, [out0], x[:, :3], 1)                # sample1 = IPA(1), written into b1's concat buffer
        out1_0 = self.level2_0(b1, precise)
        out1 = out1_0
        for layer in self.level2:
            out1 = layer(out1, precise)
        b2, _ = self._br(self.b2, [out1, out1_0], proj1, 1)                  # sample2 = IPA(2) = one more pooling of sample1
        out2_0 = self.level3_0(b2, precise)
        out2 = out2_0
        for layer in self.level3:
            out2 = layer(out2, precise)
        feat, _ = self._br(self.b3, [out2_0, out2])
        logits = Fn.EspConv.apply(feat, self.classifier.conv.weight, 1, 0, 1, precise)
        return logits, feat, out2, b2, out1, b1


def ESPNet_C(classes=19, p=2, q=8):
    return ESPNet_Encoder(classes, p, q)


class ESPNet(nn.Module):
    """The full ESPNet: ESPNet-C (`encoder.`) plus its decoder, logits at the input resolution.  H and W must be multiples of 8.

        x3 = up_l3(br(enc_logits))                                   1/8 -> 1/4; `br` is BatchNorm2d without PReLU
        y  = combine_l2_l3(cat([level3_C(b2), x3]))                  1/4: BR(2 classes) -> ESP block (2 classes -> classes, no residual)
        y  = conv(cat([up_l2(y), b1]))                               1/2: up_l2 = transposed conv + BR; conv = CBR 3x3
        logits = classifier(y)                                       1/2 -> 1/1

    The up_l3, up_l2 and classifier layers are 2x2 / stride-2 transposed convolutions without bias (`EspConvTranspose`).  forward
    returns `[logits, None, feat, out2, b2, out1, b1]` like ESPNet-C: feat (1/8) at index -5 for the pair-wise loss."""

    def __init__(self, classes=19, p=2, q=8):
        super().__init__()
        self.encoder = ESPNet_Encoder(classes, p, q)
        self.level3_C = C(128 + 3, classes, 1, 1)
        self.br = nn.BatchNorm2d(classes, eps=1e-3)
        self.conv = CBR(19 + classes, classes, 3, 1)
        self.up_l3 = nn.Sequential(nn.ConvTranspose2d(classes, classes, 2, stride=2, padding=0, output_padding=0, bias=False))
        self.combine_l2_l3 = nn.Sequential(BR(2 * classes), DilatedParllelResidualBlockB(2 * classes, classes, add=False))
        self.up_l2 = nn.Sequential(nn.ConvTranspose2d(classes, classes, 2, stride=2, padding=0, output_padding=0, bias=False),
                                   BR(classes))
        self.classifier = nn.ConvTranspose2d(classes, classes, 2, stride=2, padding=0, output_padding=0, bias=False)
        self.classes = classes

    def dropouts(self):
        return []

    def level_channels(self):
        """Widths of preds[-1] .. preds[-5], the encoder's."""
        return self.encoder.level_channels()

    def _bn(self, bn, alpha, pieces):
        return Fn.EspBnPrelu.apply(None, 0, bn.weight, bn.bias, alpha, bn.running_mean, bn.running_var, bn.num_batches_tracked,
                                   self.training, bn.momentum, bn.eps, *pieces)[0]

    def forward(self, x):
        H, W = x.shape[2], x.shape[3]
        if H % 8 or W % 8:
            raise ValueError("ESPNet needs H and W divisible by 8 (got %dx%d)" % (H, W))
        enc = self.encoder
        logits8, feat, out2, b2, out1, b1 = enc._features(x)
        c, precise = self.classes, enc.precise
        x3 = Fn.EspConvTranspose.apply(self._bn(self.br, None, [logits8[:, :c]]), self.up_l3[0].weight)              # 1/4
        l3 = Fn.EspConv.apply(b2, self.level3_C.conv.weight, 1, 0, 1, precise)
        br0 = self.combine_l2_l3[0]
        y = self._bn(br0.bn, br0.act.weight, [l3[:, :c], x3[:, :c]])
        y = self.combine_l2_l3[1](y, precise)                                                                       # 1/4
        u = Fn.EspConvTranspose.apply(y, self.up_l2[0].weight)                                                      # 1/2
        u = self._bn(self.up_l2[1].bn, self.up_l2[1].act.weight, [u[:, :c]])
        cat = Fn.EspConcat.apply(u[:, :c], b1[:, :19])
        y = Fn.EspConv.apply(cat, self.conv.conv.weight, 1, 1, 1, precise)
        y = self._bn(self.conv.bn, self.conv.act.weight, [y[:, :c]])
        logits = Fn.EspConvTranspose.apply(y, self.classifier.weight)                                               # 1/1
        return [logits[:, :c], None, feat, out2, b2[:, :131], out1, b1[:, :19]]
