"""CPU, float64: oracle/disc_pinned.py given the LeakyReLU masks the unpinned oracle/port.py chose itself reproduces port.py bit for
bit -- the outputs and attention maps of every call, the adversarial losses, the WGAN-GP value (double backward through the pinned
masks) and every parameter gradient, d / d logits of the generator pass, the BN running statistics and the spectral-norm vectors.
tests/test_disc_pinned_gpu.py then runs the same oracle with the masks the GPU kernels chose."""
import pytest
import torch

from oracle import disc_pinned, port
from test_discriminator_gpu import _size_aware_head

SHAPES = [(2, 65, 65), (1, 46, 61)]          # a 4x4 top (the reference's head) and a 2x3 top (the size-aware head)


def _port(mode):
    torch.manual_seed(11)
    Dp = port.Discriminator(mode, 19, 64)
    with torch.no_grad():
        Dp.attn1.gamma.fill_(-0.4); Dp.attn2.gamma.fill_(0.25)            # gamma = 0 would hide the attention path
        if mode == 1:
            Dp.preprocess_additional.weight.mul_(1.2)
    return Dp.double().train()


def _inputs(mode, B, H, W):
    g = torch.Generator().manual_seed(H * W + mode)
    xt = torch.randn(B, 19, H, W, generator=g, dtype=torch.float64) * 3
    xs = torch.randn(B, 19, H, W, generator=g, dtype=torch.float64) * 3
    if mode == 3:
        xs = torch.rand(B, 19, H, W, generator=g, dtype=torch.float64) * 255
    alpha = torch.rand(B, 1, 1, 1, generator=g, dtype=torch.float64)
    return xs, xt, alpha


def _record_masks(Dp):
    """forward hooks on the port's four nn.LeakyReLU: per call, the masks pre-activation > 0"""
    calls = []

    def hook(i):
        def f(module, inp, out):
            if i == 0:
                calls.append([])
            calls[-1].append(inp[0].detach() > 0)
        return f
    for i, layer in enumerate((Dp.l1, Dp.l2, Dp.l3, Dp.l4)):
        layer[1].register_forward_hook(hook(i))
    return calls


def _port_phase(Dp, xs, xt, adv, alpha):
    """The sequence of disc_pinned.discriminator_phase written with port.py's own functions."""
    xs_g = xs.clone().requires_grad_(True)
    o_g = Dp(xs_g)
    loss_g = port.adv_loss_g(o_g)
    loss_g.backward()
    for p in Dp.parameters():
        p.grad = None
    o_t, o_s = Dp(xt), Dp(xs)
    loss = port.adv_loss_d(o_s, o_t, adv)
    gp = None
    if adv == "wgan-gp":
        gp = port.gradient_penalty(Dp, xs, xt, alpha, 10.0)
        loss = loss + gp
    loss.backward()
    return dict(outs=[o_g, o_t, o_s], loss_g=loss_g, loss=loss, gp=gp, xs_grad=xs_g.grad,
                grads={n: p.grad for n, p in Dp.named_parameters() if p.grad is not None})


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


@pytest.mark.parametrize("adv", ["wgan-gp", "hinge"])
@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_pinned_oracle_is_port_bit_for_bit(shape, mode, adv):
    B, H, W = shape
    Dp = _port(mode)
    _size_aware_head(Dp, H, W)
    Dq = disc_pinned.PinnedDiscriminator(mode, 19, 64).double().train()
    Dq.load_state_dict(_port(mode).state_dict(), strict=True)
    xs, xt, alpha = _inputs(mode, B, H, W)
    masks = _record_masks(Dp)
    ref = _port_phase(Dp, xs, xt, adv, alpha)
    assert len(masks) == (4 if adv == "wgan-gp" else 3) and all(len(m) == 4 for m in masks)
    # mixed signs at every layer: the pinned factor is exercised both ways
    assert all(0 < int(m.sum()) < m.numel() for call in masks for m in call)
    hinge = None
    if adv == "hinge":
        o_t, o_s = ref["outs"][1][0].detach(), ref["outs"][2][0].detach()
        hinge = (1.0 - o_t > 0, 1.0 + o_s > 0)
    Dq.pin(masks)
    got = disc_pinned.discriminator_phase(Dq, xs, xt, adv, alpha, 10.0, hinge)
    assert Dq.pins.queue == [] and len(Dq.preacts) == len(masks)
    for c, (a, b) in enumerate(zip(got["outs"], ref["outs"])):
        for k, (ta, tb) in enumerate(zip(a, b)):
            assert _same(ta, tb), (c, k)
    for key in ("loss_g", "loss", "gp", "xs_grad"):
        if ref[key] is not None:
            assert _same(got[key], ref[key]), key
    names = {"last_conv.weight": "last.0.weight", "last_conv.bias": "last.0.bias"}
    ref_grads = {names.get(n, n): g for n, g in ref["grads"].items()}
    assert sorted(got["grads"]) == sorted(ref_grads)
    for name, g in got["grads"].items():
        assert _same(g, ref_grads[name]), name
    sp = Dp.state_dict()                                                  # running statistics, u, v after the sequence
    for name, t in Dq.state_dict().items():
        assert _same(t, sp[name if name in sp else name.replace("last.0.", "last_conv.")]), name


def test_pinning_is_live():
    """A pinned mask is what the network uses: flipping one l4 activation of the penalty's call moves the gradients (by far more
    than the last bit), and the pinned pre-activations that the mask guard reads are those of the unpinned run."""
    B, H, W = SHAPES[0]
    xs, xt, alpha = _inputs(1, B, H, W)
    runs = []
    for flip in (False, True):
        Dp = _port(1)
        masks = _record_masks(Dp)
        _port_phase(Dp, xs, xt, "wgan-gp", alpha)
        Dq = disc_pinned.PinnedDiscriminator(1, 19, 64).double().train()
        Dq.load_state_dict(_port(1).state_dict(), strict=True)
        if flip:
            z = masks[3][3]
            z.view(-1)[0] = ~z.view(-1)[0]
        Dq.pin(masks)
        runs.append(disc_pinned.discriminator_phase(Dq, xs, xt, "wgan-gp", alpha, 10.0))
        if not flip:
            for call, pre in zip(masks, Dq.preacts):
                assert all(torch.equal(m, z > 0) for m, z in zip(call, pre))
    a, b = runs[0]["grads"]["l4.0.module.weight_bar"], runs[1]["grads"]["l4.0.module.weight_bar"]
    assert float((a - b).norm() / a.norm()) > 1e-6
