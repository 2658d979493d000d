"""Float64 convolutions whose backward pass rounds its operands to TF32 as the students' backward kernels do, and the swap that puts
them into the ESPNet-C, ESPNet and MobileNetV2 ports (TEST INFRASTRUCTURE ONLY).

The students' forward convolutions are fp32-grade (3xTF32), their BatchNorm and activation kernels accumulate in double; only the
backward convolutions are TF32.  Each of them -- the data gradient on the wgmma forward kernel (or its stride-2 parity form), the
weight gradient on the wgmma wgrad kernel, both directions of the 2x2 / stride-2 transposed convolution -- reads every operand
through a TFLOAT32 tensor map, which rounds float32 to nearest with ties to even (pa_pinned.tf32_rn, DESIGN.md §4).  A product of two
TF32 values is exact in float32, so a float64 reference that rounds the same operands the same way

    dx = conv_input_grad(tf32(w), tf32(dy)),      dw = conv_weight_grad(tf32(x), tf32(dy))

leaves the kernels only their float32 accumulation and the rare TF32 rounding that flips where the kernel's float32 operand and the
reference's float64 one straddle a rounding boundary.  Operands are cast to float32 first (the kernel's storage), then rounded.

Depthwise convolutions (groups = C) are SIMT float32 kernels with double reductions and stay plain float64 autograd, as does the
students' direct SIMT route (channel counts not multiples of 4), which neither student takes (tests/test_student_blocks_float64_gpu.py
asserts it).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .pa_pinned import tf32_rn


def pin(t):
    """float64 (or float32) tensor -> float64 holding the TF32 rounding of its float32 value."""
    return tf32_rn(t.float()).double()


class _Pinned(torch.autograd.Function):
    """y = op(x, w) exactly in float64; the backward differentiates op at the pinned operands: dx from (tf32(w), tf32(dy)), dw from
    (tf32(x), tf32(dy)).  op is linear in each argument, so both gradients come from one autograd pass over the rounded values.
    pinned=False differentiates at the operands themselves (plain float64 autograd).  pinned_forward=True evaluates the forward at
    (tf32(x), tf32(w)) too, exactly in float64, as a TF32 (not 3xTF32) forward kernel reads its operands."""

    @staticmethod
    def forward(ctx, x, w, op, pinned, pinned_forward=False):
        ctx.save_for_backward(x, w)
        ctx.op, ctx.pinned = op, pinned
        return op(pin(x), pin(w)) if pinned_forward else op(x, w)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        rnd = pin if ctx.pinned else (lambda t: t.detach())
        xr, wr = rnd(x).requires_grad_(True), rnd(w).requires_grad_(True)
        with torch.enable_grad():
            y = ctx.op(xr, wr)
        dx, dw = torch.autograd.grad(y, (xr, wr), rnd(dy))
        return (dx if ctx.needs_input_grad[0] else None), (dw if ctx.needs_input_grad[1] else None), None, None, None


def conv2d(x, w, bias=None, stride=1, padding=0, dilation=1, pinned=True, pinned_forward=False):
    """F.conv2d(x, w, bias, stride, padding, dilation) in float64 with (pinned=True) the TF32-pinned backward (the bias gradient, a
    plain sum of dy, is not rounded: the kernels form it from float32 dy) and (pinned_forward=True) the TF32-pinned forward (the bias
    is added unrounded, as the kernels' epilogue adds it)."""
    def op(a, b):
        return F.conv2d(a, b, None, stride, padding, dilation)
    y = _Pinned.apply(x, w, op, pinned, pinned_forward)
    return y if bias is None else y + bias[:, None, None]


def conv_transpose2d(x, w, pinned=True):
    """F.conv_transpose2d(x, w, None, stride=2) of a (Cin, Cout, 2, 2) weight in float64 with (pinned=True) the TF32-pinned backward."""
    if tuple(w.shape[2:]) != (2, 2):
        raise ValueError("the students' transposed convolutions are 2x2 / stride 2")

    def op(a, b):
        return F.conv_transpose2d(a, b, None, stride=2)
    return _Pinned.apply(x, w, op, pinned)


class PinnedConv2d(nn.Conv2d):
    """nn.Conv2d (groups = 1) whose forward is conv2d(..., pinned=self.pinned, pinned_forward=self.pinned_forward); same parameters
    and state-dict keys."""

    pinned = True
    pinned_forward = False

    def forward(self, x):
        return conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.pinned, self.pinned_forward)


class PinnedConvTranspose2d(nn.ConvTranspose2d):
    """nn.ConvTranspose2d(k=2, stride=2, no bias) whose forward is conv_transpose2d(..., pinned=self.pinned)."""

    pinned = True

    def forward(self, x):
        return conv_transpose2d(x, self.weight, self.pinned)


def pin_convolutions(module, pinned=True):
    """Swap every nn.Conv2d / nn.ConvTranspose2d inside `module` for its pinned class in place (the depthwise ones excepted), and set
    `pinned` on every pinned convolution in it.  The swap changes the modules' class only: parameters, buffers and state-dict keys stay
    the same objects.  -> module."""
    for m in module.modules():
        if type(m) is nn.Conv2d and m.groups == 1:
            if m.padding_mode != "zeros":
                raise ValueError("the students' convolutions pad with zeros")
            m.__class__ = PinnedConv2d
        elif type(m) is nn.ConvTranspose2d:
            if m.bias is not None or m.kernel_size != (2, 2) or m.stride != (2, 2) or m.padding != (0, 0) or m.groups != 1:
                raise ValueError("the students' transposed convolutions are 2x2 / stride 2 without bias")
            m.__class__ = PinnedConvTranspose2d
        if isinstance(m, (PinnedConv2d, PinnedConvTranspose2d)):
            m.pinned = pinned
    return module
