"""oracle/student_pinned.py without a GPU: unpinned, its convolutions are float64 autograd; pinned, their gradients are float64 autograd
at operands rounded to TF32 by hand; the swap into the students' ports keeps every parameter and state-dict entry."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import espnet_full_port, espnet_port, mobilenet_port, student_pinned as sp
from oracle.pa_pinned import tf32_rn

# (n, cin, cout, h, w, k, stride, pad, dil): the students' shapes in small -- 3x3 stride 2, the ESP branches' dilations, 1x1
CONV_CASES = [(2, 5, 7, 9, 11, 3, 2, 1, 1), (1, 4, 6, 13, 10, 3, 1, 4, 4), (2, 8, 3, 7, 7, 1, 1, 0, 1), (1, 3, 4, 12, 9, 3, 1, 2, 2)]


def _data(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale


def _grads(f, x, w, dy):
    x, w = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = f(x, w)
    y.backward(dy)
    return y.detach(), x.grad, w.grad


def _hand_rounded(t):
    """float64 -> float32 -> TF32 round to nearest, ties to even, by the bit rule written out on one value at a time."""
    import struct
    out = []
    for v in t.flatten().tolist():
        u = struct.unpack("<I", struct.pack("<f", v))[0]
        low, keep = u & 0x1FFF, u & ~0x1FFF
        if low > 0x1000 or (low == 0x1000 and (u >> 13) & 1):
            keep += 0x2000
        out.append(struct.unpack("<f", struct.pack("<I", keep & 0xFFFFFFFF))[0])
    return torch.tensor(out, dtype=torch.float64).view(t.shape)


@pytest.mark.parametrize("case", CONV_CASES, ids=repr)
def test_unpinned_conv2d_is_float64_autograd(case):
    n, cin, cout, h, w, k, s, p, d = case
    x, wt = _data((n, cin, h, w), 1), _data((cout, cin, k, k), 2, 0.3)
    y0 = F.conv2d(x, wt, None, s, p, d)
    dy = _data(y0.shape, 3)
    got = _grads(lambda a, b: sp.conv2d(a, b, None, s, p, d, pinned=False), x, wt, dy)
    ref = _grads(lambda a, b: F.conv2d(a, b, None, s, p, d), x, wt, dy)
    for g, r in zip(got, ref):
        torch.testing.assert_close(g, r, rtol=1e-13, atol=1e-13)


def test_unpinned_conv_transpose2d_is_float64_autograd():
    x, wt = _data((2, 5, 4, 6), 4), _data((5, 7, 2, 2), 5, 0.3)
    dy = _data((2, 7, 8, 12), 6)
    got = _grads(lambda a, b: sp.conv_transpose2d(a, b, pinned=False), x, wt, dy)
    ref = _grads(lambda a, b: F.conv_transpose2d(a, b, None, stride=2), x, wt, dy)
    for g, r in zip(got, ref):
        torch.testing.assert_close(g, r, rtol=1e-13, atol=1e-13)


def test_unpinned_functions_pass_gradcheck():
    x = _data((1, 3, 6, 5), 7).requires_grad_(True)
    w = _data((4, 3, 3, 3), 8).requires_grad_(True)
    b = _data((4,), 9).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, c, e: sp.conv2d(a, c, e, 2, 2, 2, pinned=False), (x, w, b))
    xt = _data((1, 4, 3, 2), 10).requires_grad_(True)
    wt = _data((4, 3, 2, 2), 11).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, c: sp.conv_transpose2d(a, c, pinned=False), (xt, wt))


def test_pin_is_the_hand_rounding():
    """pin() is float32 then TF32 RNE: checked against the rule applied bit by bit, at random values and at exact ties both ways."""
    v = _data((257,), 12, 3.0)
    ties = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -11 + 2.0 ** -20], dtype=torch.float64)
    for t in (v, ties):
        assert torch.equal(sp.pin(t), _hand_rounded(t))
    assert sp.pin(ties).tolist() == [1.0, 1.0 + 2.0 ** -9, -1.0, 1.0 + 2.0 ** -10]


@pytest.mark.parametrize("case", CONV_CASES, ids=repr)
def test_pinned_conv2d_gradients_are_autograd_at_rounded_operands(case):
    n, cin, cout, h, w, k, s, p, d = case
    x, wt = _data((n, cin, h, w), 13), _data((cout, cin, k, k), 14, 0.3)
    b = _data((cout,), 15)
    dy = _data(F.conv2d(x, wt, None, s, p, d).shape, 16)
    xb, wb, bb = x.clone().requires_grad_(True), wt.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = sp.conv2d(xb, wb, bb, s, p, d, pinned=True)
    y.backward(dy)
    # forward exact float64
    torch.testing.assert_close(y.detach(), F.conv2d(x, wt, b, s, p, d), rtol=1e-13, atol=1e-13)
    xr, wr, dyr = _hand_rounded(x), _hand_rounded(wt), _hand_rounded(dy)
    dx_ref = torch.nn.grad.conv2d_input(x.shape, wr, dyr, s, p, d)
    dw_ref = torch.nn.grad.conv2d_weight(xr, wt.shape, dyr, s, p, d)
    torch.testing.assert_close(xb.grad, dx_ref, rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(wb.grad, dw_ref, rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(bb.grad, dy.sum((0, 2, 3)), rtol=1e-13, atol=1e-13)
    # the rounding is visible: the pinned gradients are not the unpinned ones
    assert (xb.grad - torch.nn.grad.conv2d_input(x.shape, wt, dy, s, p, d)).abs().max() > 1e-6


def test_pinned_conv_transpose2d_gradients_are_autograd_at_rounded_operands():
    x, wt = _data((2, 6, 3, 5), 17), _data((6, 5, 2, 2), 18, 0.3)
    dy = _data((2, 5, 6, 10), 19)
    got = _grads(lambda a, b: sp.conv_transpose2d(a, b, pinned=True), x, wt, dy)
    xr, wr, dyr = _hand_rounded(x), _hand_rounded(wt), _hand_rounded(dy)
    _, dx_ref, _ = _grads(lambda a, b: F.conv_transpose2d(a, b, None, stride=2), x, wr, dyr)
    _, _, dw_ref = _grads(lambda a, b: F.conv_transpose2d(a, b, None, stride=2), xr, wt, dyr)
    torch.testing.assert_close(got[0], F.conv_transpose2d(x, wt, None, stride=2), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(got[1], dx_ref, rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(got[2], dw_ref, rtol=1e-13, atol=1e-13)


def _ported_blocks():
    enc = espnet_port.build_student(3)
    full = espnet_full_port.build_student(4, classes=11)
    mb = mobilenet_port.build_student(5)
    return [("DownSamplerB", enc.level2_0), ("DilatedParllelResidualBlockB", enc.level3[0]),
            ("DilatedParllelResidualBlockB add=False", full.combine_l2_l3[1]), ("decoder", full),
            ("InvertedResidual t=1", mb.features[1]), ("InvertedResidual", mb.features[4]), ("MobileNetV2", mb)]


@pytest.mark.parametrize("name,block", _ported_blocks(), ids=lambda v: v if isinstance(v, str) else "")
def test_swap_keeps_state_dict_and_parameters(name, block):
    before = {k: (v, v.clone()) for k, v in block.state_dict(keep_vars=True).items()}
    params = dict(block.named_parameters())
    n_dw = sum(1 for m in block.modules() if type(m) is nn.Conv2d and m.groups > 1)
    sp.pin_convolutions(block)
    after = block.state_dict(keep_vars=True)
    assert list(after) == list(before)
    for k, v in after.items():
        assert v is before[k][0] and torch.equal(v, before[k][1]), k
    assert dict(block.named_parameters()) == params
    kinds = [type(m) for m in block.modules()]
    assert nn.ConvTranspose2d not in kinds
    assert sum(1 for t in kinds if t is nn.Conv2d) == n_dw                      # only the depthwise convolutions stay plain
    assert any(isinstance(m, (sp.PinnedConv2d, sp.PinnedConvTranspose2d)) for m in block.modules())


def test_swapped_block_runs_pinned_and_unpinned():
    """A swapped InvertedResidual in float64: forward equals the unswapped one; unpinned gradients equal plain autograd, pinned ones
    differ from them by TF32 rounding only (relative 1e-6 .. 1e-2)."""
    torch.manual_seed(0)
    ref = mobilenet_port.build_student(6).features[2].double().train()
    x = _data((2, 16, 10, 12), 20)
    import copy
    outs = {}
    for mode in ("plain", False, True):
        m = copy.deepcopy(ref)
        if mode != "plain":
            sp.pin_convolutions(m, pinned=mode)
        xb = x.clone().requires_grad_(True)
        y = m(xb)
        y.backward(_data(y.shape, 21))
        outs[mode] = (y.detach(), xb.grad, [p.grad for p in m.parameters()])
    for a, b in zip(outs["plain"][:2], outs[False][:2]):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
    for a, b in zip(outs["plain"][2], outs[False][2]):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(outs["plain"][0], outs[True][0], rtol=1e-12, atol=1e-12)
    rel = float((outs[True][1] - outs["plain"][1]).norm() / outs["plain"][1].norm())
    assert 1e-6 < rel < 1e-2, rel
