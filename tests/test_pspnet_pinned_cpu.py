"""oracle/pspnet_pinned.py without a GPU: unpinned, its convolutions are float64 autograd; forward- and backward-pinned, they are
float64 autograd at operands rounded to TF32 by hand; a mask taken from the float64 sign gives the unpinned port; the swap keeps every
parameter and state-dict entry of the ResNet18 and ResNet101 ports; which forwards are pinned follows the product module."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import port, pspnet_pinned as pp, student_pinned as sp
from test_student_pinned_cpu import CONV_CASES, _data, _hand_rounded


@pytest.mark.parametrize("case", CONV_CASES, ids=repr)
def test_unpinned_conv_is_float64_autograd(case):
    n, cin, cout, h, w, k, s, p, d = case
    x, wt, b = _data((n, cin, h, w), 1), _data((cout, cin, k, k), 2, 0.3), _data((cout,), 3)
    y0 = F.conv2d(x, wt, b, s, p, d)
    dy = _data(y0.shape, 4)
    got, ref = [], []
    for f, out in ((lambda a, c, e: sp.conv2d(a, c, e, s, p, d, pinned=False, pinned_forward=False), got),
                   (lambda a, c, e: F.conv2d(a, c, e, s, p, d), ref)):
        xa, wa, ba = (t.clone().requires_grad_(True) for t in (x, wt, b))
        y = f(xa, wa, ba)
        y.backward(dy)
        out += [y.detach(), xa.grad, wa.grad, ba.grad]
    for g, r in zip(got, ref):
        torch.testing.assert_close(g, r, rtol=1e-13, atol=1e-13)
    xg, wg, bg = (t[:1, :2, :5, :5].clone().requires_grad_(True) if t.dim() == 4 else t.clone().requires_grad_(True)
                  for t in (x, wt[:, :2], b))
    assert torch.autograd.gradcheck(lambda a, c, e: sp.conv2d(a, c, e, s, p, d, pinned=False), (xg, wg, bg))


@pytest.mark.parametrize("case", CONV_CASES, ids=repr)
def test_forward_and_backward_pinned_conv_is_autograd_at_rounded_operands(case):
    """y = conv(tf32(x), tf32(w)) + b exactly; dx from (tf32(w), tf32(dy)), dw from (tf32(x), tf32(dy)); db = sum dy unrounded.  The
    operands carry exact ties (float32 values halfway between two TF32 values) both ways."""
    n, cin, cout, h, w, k, s, p, d = case
    x, wt, b = _data((n, cin, h, w), 5), _data((cout, cin, k, k), 6, 0.3), _data((cout,), 7)
    x.view(-1)[:4] = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11), 0.5 + 2.0 ** -12], dtype=torch.float64)
    wt.view(-1)[:2] = torch.tensor([0.25 + 2.0 ** -13, -(0.25 + 3 * 2.0 ** -13)], dtype=torch.float64)
    dy = _data(F.conv2d(x, wt, None, s, p, d).shape, 8)
    dy.view(-1)[:2] = torch.tensor([2.0 + 2.0 ** -10, -(2.0 + 3 * 2.0 ** -10)], dtype=torch.float64)
    xa, wa, ba = (t.clone().requires_grad_(True) for t in (x, wt, b))
    y = sp.conv2d(xa, wa, ba, s, p, d, pinned=True, pinned_forward=True)
    y.backward(dy)
    xr, wr, dyr = _hand_rounded(x), _hand_rounded(wt), _hand_rounded(dy)
    torch.testing.assert_close(y.detach(), F.conv2d(xr, wr, b, s, p, d), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(xa.grad, torch.nn.grad.conv2d_input(x.shape, wr, dyr, s, p, d), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(wa.grad, torch.nn.grad.conv2d_weight(xr, wt.shape, dyr, s, p, d), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(ba.grad, dy.sum((0, 2, 3)), rtol=1e-13, atol=1e-13)
    # the forward rounding is visible, and the ties went to even
    assert (y.detach() - F.conv2d(x, wt, b, s, p, d)).abs().max() > 1e-6
    assert xr.view(-1)[:4].tolist() == [1.0, 1.0 + 2.0 ** -9, -1.0, 0.5]


def _net(arch, seed=0, classes=5):
    torch.manual_seed(seed)
    net = port.PSPNet(arch, classes)
    port.perturb_bn_stats(net, seed + 1)
    return net


@pytest.mark.parametrize("arch", ["resnet18", "resnet101"])
def test_swap_keeps_state_dict_and_parameters(arch):
    net = _net(arch)
    before = {k: (v, v.clone()) for k, v in net.state_dict(keep_vars=True).items()}
    params = dict(net.named_parameters())
    n_conv = sum(1 for m in net.modules() if type(m) is torch.nn.Conv2d)
    pp.pin_pspnet(net)
    after = net.state_dict(keep_vars=True)
    assert list(after) == list(before)
    for k, v in after.items():
        assert v is before[k][0] and torch.equal(v, before[k][1]), k
    assert dict(net.named_parameters()) == params
    kinds = [type(m) for m in net.modules()]
    assert torch.nn.Conv2d not in kinds and port.ABN not in kinds and port._Basic not in kinds
    assert kinds.count(sp.PinnedConv2d) == n_conv
    acts = pp.pinned_acts(net)
    leaky = 5                                                           # four PSP stages and the PSP bottleneck ... and the DSN
    assert sum(isinstance(m, pp.PinnedABN) for m in acts.values()) == leaky + 1
    assert sum(isinstance(m, pp.PinnedAct) for m in acts.values()) == 2 + (8 if arch == "resnet18" else 0)


def _product(arch, classes=5):
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Bottleneck, Res_pspnet
    return Res_pspnet(BasicBlock, [2, 2, 2, 2], classes) if arch == "resnet18" else Res_pspnet(Bottleneck, [3, 4, 23, 3], classes)


@pytest.mark.parametrize("arch", ["resnet18", "resnet101"])
def test_forward_pinning_follows_the_product_module(arch):
    """Frozen: every forward pinned.  Training: exactly the convolutions the product runs in TF32 -- precise unset (layer3, layer4,
    PSP, DSN, head) or a channel count that is not a multiple of 4; the stem's small-Cin route and the other precise ones are 3xTF32."""
    prod = _product(arch)
    mods = dict(prod.named_modules())
    for frozen in (True, False):
        net = pp.pin_pspnet(_net(arch), prod, frozen=frozen)
        convs = {n: m for n, m in net.named_modules() if isinstance(m, sp.PinnedConv2d)}
        for n, m in convs.items():
            early = n.startswith(("conv", "layer1", "layer2"))
            assert mods[n].precise == early, n
            assert m.pinned_forward == (frozen or not early), n
            assert m.pinned
    prod.conv2.precise = True
    prod.conv2.weight = torch.nn.Parameter(torch.zeros(64, 6, 3, 3))       # Cin 6: Fn.Conv2d's padded TF32 route
    assert pp.tf32_forward(prod.conv2, False) and not pp.tf32_forward(prod.conv3, False)
    assert pp.tf32_forward(prod.conv3, False, pitch=132) and not pp.tf32_forward(prod.conv1, False)
    assert not pp.pin_pspnet(_net(arch), pinned=False).conv3.pinned


def _close(a, b):
    """Equal to float64 rounding: within 1e-11 of the tensor's largest element, or of 1 for the analytically zero gradient of the DSN
    convolution's bias (cancellation residue near 1e-16)."""
    assert float((a - b).abs().max()) <= 1e-11 * max(float(b.abs().max()), 1.0)


def _run(net, x, dy_seed, masks=None):
    for name, m in pp.pinned_acts(net).items():
        m.mask = None if masks is None else masks.get(name)
    xa = x.clone().requires_grad_(True)
    outs = net(xa)
    loss = sum((o * _data(o.shape, dy_seed + i)).sum() for i, o in enumerate(outs))
    loss.backward()
    return [o.detach() for o in outs], xa.grad, {n: p.grad.clone() for n, p in net.named_parameters()}


@pytest.mark.parametrize("arch", ["resnet18", "resnet101"])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_masks_from_the_float64_sign_reproduce_the_port(arch, training):
    """The unpinned network without masks is the port (to 1e-11 of each tensor's largest element: the pinned convolution adds its bias after the convolution); with
    every mask set from the float64 pre-activation's sign it is again the port -- bit for bit against the unmasked swap through the
    ReLUs, to the same through the leaky ABNs, whose port backward recovers z as y / slope."""
    torch.manual_seed(3)
    base = _net(arch, 2).double().train(training)
    for d, c in zip(base.dropouts(), (base.pspmodule.bottleneck[0].out_channels, base.dsn[0].out_channels)):
        d.injected = (torch.rand(2, c) >= d.p).double()
    x = _data((2, 3, 33, 41), 9)
    want = _run(copy.deepcopy(base), x, 20)
    net = pp.pin_pspnet(copy.deepcopy(base), pinned=False)
    unmasked = got = _run(net, x, 20)
    for a, b in zip(got[0] + [got[1]], want[0] + [want[1]]):
        _close(a, b)
    for k in want[2]:
        _close(got[2][k], want[2][k])
    masks = {n: (m.z > 0 if isinstance(m, pp.PinnedAct) else m.z >= 0) for n, m in pp.pinned_acts(net).items()}
    assert len(masks) == 6 + (10 if arch == "resnet18" else 2)
    net = pp.pin_pspnet(copy.deepcopy(base), pinned=False)
    got = _run(net, x, 20, masks)
    for a, b in zip(got[0] + [got[1]], want[0] + [want[1]]):
        _close(a, b)
    for k in want[2]:
        _close(got[2][k], want[2][k])
    relu = [n for n, m in pp.pinned_acts(net).items() if isinstance(m, pp.PinnedAct)]
    assert relu
    for n, m in pp.pinned_acts(net).items():
        assert m.z is not None and torch.equal(m.z > 0 if n in relu else m.z >= 0, masks[n]), n
    # bit for bit where only ReLU masks are set
    net = pp.pin_pspnet(copy.deepcopy(base), pinned=False)
    got = _run(net, x, 20, {n: masks[n] for n in relu})
    for a, b in zip(got[0] + [got[1]], unmasked[0] + [unmasked[1]]):
        assert torch.equal(a, b)
    for k in want[2]:
        assert torch.equal(got[2][k], unmasked[2][k]), k
