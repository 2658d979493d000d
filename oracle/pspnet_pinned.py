"""The PSPNet / dilated-ResNet port (oracle/port.PSPNet) with the TF32 operands of its convolutions and the masks of its inner
activations pinned as the product computes them (TEST INFRASTRUCTURE ONLY).

Three kinds of pinning, each switchable, all in float64:

  * Backward convolutions (every one in the product is TF32): oracle/student_pinned.py's, dx from (tf32(w), tf32(dy)) and dw from
    (tf32(x), tf32(dy)); the bias gradient is a plain sum.
  * Forward convolutions that the product runs in TF32 rather than 3xTF32: y = conv(tf32(x), tf32(w)) exactly, the bias added
    unrounded.  Which ones those are is read off the product module (`tf32_forward`), never listed here: the `frozen` path runs every
    convolution in TF32; the training path runs a convolution in 3xTF32 only when its `precise` flag is set and Fn.Conv2d.forward
    takes a 3xTF32 route -- the small-Cin im2col route of the stem, or the padded route when Cin and Cout are multiples of 4 and the
    input's pitch equals its channel count.
  * Activations inside a block: the ReLU after `bn1` of a BasicBlock and after `bn1` / `bn2` of the stem (`PinnedAct` modules), and
    the LeakyReLU of every leaky ABN (`PinnedABN`, used on the PSP stages and the DSN).  Given a boolean `mask` (taken from the
    product's own float32 output of that activation) the activation is z * where(mask, 1, slope), so that the reference evaluates
    the product's linear piece: a pre-activation within float32 rounding of 0 then cannot move a gradient by O(1).  Every call
    records its pre-activation in `z`, from which a caller counts where the mask disagrees
    with the float64 sign.  Without a mask the activation is the port's.

`pin_pspnet` swaps these classes into a port network in place; parameters, buffers and state-dict keys stay the same objects.
PinnedPSPNet.stem runs conv1-3 alone, so that a caller can run the network stage by stage.
tests/test_pspnet_pinned_cpu.py checks all of this on the CPU.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import port
from .student_pinned import PinnedConv2d


def tf32_forward(conv, frozen, pitch=None):
    """Whether the product convolution module `conv` (networks/pspnet_combine.Conv2d) runs its forward in plain TF32: always on the
    `frozen` path; on the training path unless `precise` selects a 3xTF32 route of Fn.Conv2d.forward (`pitch`: the input's pixel
    pitch, its channel count by default)."""
    from structure_knowledge_distillation_b200 import functions as Fn
    if frozen or not conv.precise:
        return True
    w = conv.weight
    if Fn._small_cin(w) and conv.bias is None:
        return False                                          # im2col + 3xTF32 (the stem's conv1; its input never requires grad)
    cout, cin = w.shape[0], w.shape[1]
    return not (cout % 4 == 0 and cin % 4 == 0 and (pitch is None or pitch == cin))


class PinnedAct(nn.Module):
    """ReLU (slope 0) or LeakyReLU(slope) with an optional pinned mask: z * where(mask, 1, slope).  No parameters or buffers."""

    def __init__(self, slope=0.0):
        super().__init__()
        self.slope, self.mask, self.z = slope, None, None

    def forward(self, z):
        self.z = z.detach()
        if self.mask is None:
            return F.relu(z) if self.slope == 0 else F.leaky_relu(z, self.slope)
        if self.mask.shape != z.shape:
            raise ValueError("pinned mask %s does not match pre-activation %s" % (tuple(self.mask.shape), tuple(z.shape)))
        return z * torch.where(self.mask.to(z.device), z.new_tensor(1.0), z.new_tensor(self.slope))


class PinnedABN(port.ABN):
    """port.ABN whose leaky activation takes a pinned mask (`mask`, `z` as PinnedAct's).  Without a mask it is port.ABN itself; with
    one it is the activation-free ABN followed by the masked activation."""

    mask = None
    z = None

    def forward(self, x):
        if self.mask is None or self.activation != port.ACT_LEAKY:
            y = super().forward(x)
            if self.activation == port.ACT_LEAKY:
                self.z = torch.where(y < 0, y / self.slope, y).detach()     # as port._ABNFn.backward recovers it
            return y
        z = port._ABNFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.training, self.momentum, self.eps,
                              port.ACT_NONE, self.slope)
        self.z = z.detach()
        if self.mask.shape != z.shape:
            raise ValueError("pinned mask %s does not match pre-activation %s" % (tuple(self.mask.shape), tuple(z.shape)))
        return z * torch.where(self.mask.to(z.device), z.new_tensor(1.0), z.new_tensor(self.slope))


class PinnedBasic(port._Basic):
    """port._Basic with its inner ReLU (after bn1) a PinnedAct `act1`."""

    def forward(self, x):
        r = x if self.downsample is None else self.downsample(x)
        o = self.act1(self.bn1(self.conv1(x)))
        o = self.bn2(self.conv2(o))
        return F.relu(o + r)


class PinnedPSPNet(port.PSPNet):
    """port.PSPNet with the stem's inner ReLUs PinnedActs `act1`, `act2`."""

    def forward(self, x):
        x1, x2, x3 = self.backbone(x)
        x_dsn = self.dsn(x3)
        x4 = self.layer4(x3)
        feat = self.pspmodule(x4)
        return [self.head(feat), x_dsn, feat, x4, x3, x2, x1]

    def stem(self, x):
        """conv1-3 with their ABN + ReLU, before the max-pool."""
        x = self.act1(self.bn1(self.conv1(x)))
        x = self.act2(self.bn2(self.conv2(x)))
        return F.relu(self.bn3(self.conv3(x)))

    def backbone(self, x):
        x1 = self.layer1(self.maxpool(self.stem(x)))
        x2 = self.layer2(x1)
        return x1, x2, self.layer3(x2)


def pin_pspnet(net, prod=None, pinned=True, frozen=False):
    """Swap the pinned classes into the port network `net` (port.PSPNet) in place -> net.

    pinned: every convolution's backward is TF32-pinned (False: plain float64 autograd).  prod: the product network with the same
    state-dict keys; each convolution's forward is pinned where tf32_forward(its product module, frozen) says so (prod None: no forward
    is pinned).  Masks start unset (the port's activations)."""
    if not isinstance(net, port.PSPNet):
        raise TypeError("pin_pspnet takes a port.PSPNet")
    prod_mods = dict(prod.named_modules()) if prod is not None else {}
    if not isinstance(net, PinnedPSPNet):
        net.__class__ = PinnedPSPNet
        net.act1, net.act2 = PinnedAct(), PinnedAct()
    for name, m in list(net.named_modules()):
        if type(m) is nn.Conv2d:
            if m.groups != 1 or m.padding_mode != "zeros":
                raise ValueError("the PSPNet convolutions are dense and pad with zeros")
            m.__class__ = PinnedConv2d
        elif type(m) is port.ABN:
            m.__class__ = PinnedABN
        elif type(m) is port._Basic:
            m.__class__ = PinnedBasic
            m.act1 = PinnedAct()
        if isinstance(m, PinnedConv2d):
            m.pinned = pinned
            m.pinned_forward = bool(prod is not None and tf32_forward(prod_mods[name], frozen))
    return net


def pinned_acts(net):
    """{module path: PinnedAct / leaky PinnedABN} of a pin_pspnet network: every activation that takes a mask."""
    return {n: m for n, m in net.named_modules()
            if isinstance(m, PinnedAct) or (isinstance(m, PinnedABN) and m.activation == port.ACT_LEAKY)}


def clear_masks(net):
    for m in pinned_acts(net).values():
        m.mask, m.z = None, None
