"""The SAGAN discriminator of oracle/port.py with its LeakyReLU masks pinned (TEST INFRASTRUCTURE ONLY).

A LeakyReLU network is piecewise smooth: inside one piece every LeakyReLU multiplies its input by a fixed 1 or 0.1.  Where the
fp32 kernels and a float64 oracle round a pre-activation to opposite sides of zero they evaluate different pieces, and every
gradient below that activation moves by about 5e-3 (tests/test_discriminator_gpu.py).  Run with the masks the GPU chose, this
oracle evaluates the GPU's piece, so its values, first derivatives and -- through autograd's double backward, a pinned mask being
piecewise constant -- the WGAN-GP's second derivatives are what the kernels should produce up to their own rounding.

  * `PinnedDiscriminator` is port.Discriminator (same constructor, parameters, buffers and state-dict names, same spectral-norm
    power iteration) whose l1..l4 LeakyReLUs read one mask per layer and per call from a queue (`pin`).  A call with no queued
    masks is the unpinned port.  Every call records its four pre-activations in `preacts`.
  * Its head is size-aware like the product's: a map smaller than 4x4 meets the top-left window of the 4x4 kernel (the logits of
    360x480 crops end in a 2x3 map).  On maps of 4x4 and more it is the port's nn.Conv2d.
  * `adv_loss_d` / `gradient_penalty` are port.adv_loss_d / port.gradient_penalty with the hinge's relu masks pinned the same way
    and the penalty's per-image gradient norms returned.

tests/test_disc_pinned_cpu.py checks that with the masks the unpinned port chose itself, all of this is port.py bit for bit.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import port

SLOPE = 0.1


class _Pins:
    """Mask queue and pre-activation record shared by the four pinned LeakyReLUs of one discriminator."""

    def __init__(self):
        self.queue = []          # per call: list of 4 boolean masks shaped like the pre-activations, or None (unpinned)
        self.current = None
        self.preacts = []        # per call: the 4 pre-activations it met

    def begin_call(self):
        self.current = self.queue.pop(0) if self.queue else None
        self.preacts.append([])


class PinnedLeakyReLU(nn.Module):
    """LeakyReLU(0.1) whose mask is given: z * where(mask, 1, 0.1).  Without a mask it is nn.LeakyReLU(0.1)."""

    def __init__(self, pins, index):
        super().__init__()
        self.pins, self.index = pins, index

    def forward(self, z):
        pins = self.pins
        pins.preacts[-1].append(z.detach())
        if pins.current is None:
            return F.leaky_relu(z, SLOPE)
        mask = pins.current[self.index]
        if mask.shape != z.shape:
            raise ValueError("pinned mask %s does not match pre-activation %s" % (tuple(mask.shape), tuple(z.shape)))
        return z * torch.where(mask.to(z.device), z.new_tensor(1.0), z.new_tensor(SLOPE))


class SizeAwareHead(nn.Conv2d):
    """The 4x4 "last" convolution; on a map smaller than 4x4 it uses the top-left min(4, H) x min(4, W) window of its kernel."""

    def forward(self, x):
        kh, kw = min(4, x.shape[2]), min(4, x.shape[3])
        if (kh, kw) == (4, 4):
            return super().forward(x)
        return F.conv2d(x, self.weight[:, :, :kh, :kw], self.bias)


class PinnedDiscriminator(port.Discriminator):
    def __init__(self, preprocess_mode=1, in_ch=19, conv_dim=64):
        super().__init__(preprocess_mode, in_ch, conv_dim)
        self.pins = _Pins()
        for i, layer in enumerate((self.l1, self.l2, self.l3, self.l4)):
            layer[1] = PinnedLeakyReLU(self.pins, i)
        head = SizeAwareHead(8 * conv_dim, 1, 4)
        head.load_state_dict(self.last[0].state_dict())
        self.last[0] = head

    def pin(self, calls):
        """Queue masks for the next calls, in call order: each entry is a list of the 4 layers' boolean masks (NCHW, the shape
        of the pre-activation) or None for an unpinned call."""
        self.pins.queue.extend(calls)

    @property
    def preacts(self):
        return self.pins.preacts

    def forward(self, x):
        self.pins.begin_call()
        return super().forward(x)


def adv_loss_d(d_out_S, d_out_T, adv_type, hinge_masks=None):
    """port.adv_loss_d; for hinge with hinge_masks = (1 - real > 0, 1 + fake > 0) the relus become products with those masks."""
    if adv_type != "hinge" or hinge_masks is None:
        return port.adv_loss_d(d_out_S, d_out_T, adv_type)
    real, fake = d_out_T[0], d_out_S[0]
    m_real, m_fake = (m.to(device=real.device, dtype=real.dtype) for m in hinge_masks)
    return ((1.0 - real) * m_real).mean() + ((1.0 + fake) * m_fake).mean()


def gradient_penalty(D, logits_S, logits_T, alpha, lambda_gp):
    """port.gradient_penalty -> (penalty, per-image norms of d sum D(x) / dx)."""
    x = (alpha * logits_T.detach() + (1 - alpha) * logits_S.detach()).requires_grad_(True)
    out = D(x)[0]
    (g,) = torch.autograd.grad(out, x, torch.ones_like(out), create_graph=True, retain_graph=True)
    gn = g.flatten(1).pow(2).sum(1).sqrt()
    return lambda_gp * ((gn - 1) ** 2).mean(), gn


def discriminator_phase(D, xs, xt, adv_type, alpha, lambda_gp=10.0, hinge_masks=None):
    """NetModel's uses of D in one step (networks/kd_model.py): the generator pass -mean D(xs) with d / d xs, then with fresh
    gradients D(xt), D(xs), the adversarial loss (+ the penalty at alpha xt + (1 - alpha) xs for wgan-gp) and its backward.
    Returns the outputs of the three calls, the losses, the penalty and its norms, d / d xs of the generator pass and every
    parameter gradient by name."""
    xs_g = xs.detach().clone().requires_grad_(True)
    o_g = D(xs_g)
    loss_g = port.adv_loss_g(o_g)
    loss_g.backward()
    for p in D.parameters():
        p.grad = None
    o_t = D(xt)
    o_s = D(xs)
    loss = adv_loss_d(o_s, o_t, adv_type, hinge_masks)
    gp = norms = None
    if adv_type == "wgan-gp":
        gp, norms = gradient_penalty(D, xs, xt, alpha, lambda_gp)
        loss = loss + gp
    loss.backward()
    return dict(outs=[o_g, o_t, o_s], loss_g=loss_g, loss=loss, gp=gp, norms=norms, xs_grad=xs_g.grad,
                grads={n: p.grad for n, p in D.named_parameters() if p.grad is not None})
