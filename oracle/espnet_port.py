"""ESPNet-C (Mehta et al., ECCV 2018, the encoder-only ESPNet) in plain torch -- nn.Conv2d, nn.BatchNorm2d, nn.PReLU, nn.AvgPool2d,
torch.cat -- and the distillation step with it as the student.  TEST INFRASTRUCTURE ONLY: the CPU restatement the sm_90a student
(structure_knowledge_distillation_b200/networks/espnet.py) is checked against.  The reference ships no ESPNet source, so the
architecture is the one the package documents (same attribute names, hence the same state-dict keys).

Step decisions (no reference exists for them):
  * the teacher (PSPNet, ceil-mode stem pool) is on 46x61 at 360x480 where ESPNet-C is on 45x60: the two teacher tensors the
    distillation terms read, preds_T[0] and preds_T[-5], are resized to the student's grid with bilinear align_corners=True;
  * the task loss is a single cross entropy (ESPNet-C has no auxiliary head): CE(up(logits)), bilinear align_corners, ignore 255.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import port


class CBR(nn.Module):
    def __init__(self, nIn, nOut, kSize, stride=1):
        super().__init__()
        self.conv = nn.Conv2d(nIn, nOut, kSize, stride, (kSize - 1) // 2, bias=False)
        self.bn = nn.BatchNorm2d(nOut, eps=1e-3)
        self.act = nn.PReLU(nOut)

    def forward(self, x):
        return self.act(self.bn(self.conv(x)))


class BR(nn.Module):
    def __init__(self, nOut):
        super().__init__()
        self.bn = nn.BatchNorm2d(nOut, eps=1e-3)
        self.act = nn.PReLU(nOut)

    def forward(self, x):
        return self.act(self.bn(x))


class C(nn.Module):
    def __init__(self, nIn, nOut, kSize, stride=1):
        super().__init__()
        self.conv = nn.Conv2d(nIn, nOut, kSize, stride, (kSize - 1) // 2, bias=False)

    def forward(self, x):
        return self.conv(x)


class CDilated(nn.Module):
    def __init__(self, nIn, nOut, kSize, stride=1, d=1):
        super().__init__()
        self.conv = nn.Conv2d(nIn, nOut, kSize, stride, (kSize - 1) // 2 * d, bias=False, dilation=d)

    def forward(self, x):
        return self.conv(x)


def _esp(m, x):
    o = m.c1(x)
    d1 = m.d1(o)
    a1 = m.d2(o)
    a2 = a1 + m.d4(o)
    a3 = a2 + m.d8(o)
    a4 = a3 + m.d16(o)
    return torch.cat([d1, a1, a2, a3, a4], 1)


class DownSamplerB(nn.Module):
    def __init__(self, nIn, nOut):
        super().__init__()
        n = nOut // 5
        n1 = nOut - 4 * n
        self.c1 = C(nIn, n, 3, 2)
        self.d1 = CDilated(n, n1, 3, 1, 1)
        self.d2 = CDilated(n, n, 3, 1, 2)
        self.d4 = CDilated(n, n, 3, 1, 4)
        self.d8 = CDilated(n, n, 3, 1, 8)
        self.d16 = CDilated(n, n, 3, 1, 16)
        self.bn = nn.BatchNorm2d(nOut, eps=1e-3)
        self.act = nn.PReLU(nOut)

    def forward(self, x):
        return self.act(self.bn(_esp(self, x)))


class DilatedParllelResidualBlockB(nn.Module):
    def __init__(self, nIn, nOut, add=True):
        super().__init__()
        n = nOut // 5
        n1 = nOut - 4 * n
        self.c1 = C(nIn, n, 1, 1)
        self.d1 = CDilated(n, n1, 3, 1, 1)
        self.d2 = CDilated(n, n, 3, 1, 2)
        self.d4 = CDilated(n, n, 3, 1, 4)
        self.d8 = CDilated(n, n, 3, 1, 8)
        self.d16 = CDilated(n, n, 3, 1, 16)
        self.bn = BR(nOut)
        self.add = add

    def forward(self, x):
        combine = _esp(self, x)
        if self.add:
            combine = x + combine
        return self.bn(combine)


class InputProjectionA(nn.Module):
    def __init__(self, samplingTimes):
        super().__init__()
        self.pool = nn.ModuleList([nn.AvgPool2d(3, stride=2, padding=1) for _ in range(samplingTimes)])

    def forward(self, x):
        for p in self.pool:
            x = p(x)
        return x


class ESPNet_Encoder(nn.Module):
    def __init__(self, classes=19, p=2, q=8):
        super().__init__()
        self.level1 = CBR(3, 16, 3, 2)
        self.sample1 = InputProjectionA(1)
        self.sample2 = InputProjectionA(2)
        self.b1 = BR(16 + 3)
        self.level2_0 = DownSamplerB(16 + 3, 64)
        self.level2 = nn.ModuleList([DilatedParllelResidualBlockB(64, 64) for _ in range(p)])
        self.b2 = BR(128 + 3)
        self.level3_0 = DownSamplerB(128 + 3, 128)
        self.level3 = nn.ModuleList([DilatedParllelResidualBlockB(128, 128) for _ in range(q)])
        self.b3 = BR(256)
        self.classifier = C(256, classes, 1, 1)

    def forward(self, x):
        out0 = self.level1(x)
        inp1 = self.sample1(x)
        inp2 = self.sample2(x)
        b1 = self.b1(torch.cat([out0, inp1], 1))
        out1_0 = self.level2_0(b1)
        out1 = out1_0
        for layer in self.level2:
            out1 = layer(out1)
        b2 = self.b2(torch.cat([out1, out1_0, inp2], 1))
        out2_0 = self.level3_0(b2)
        out2 = out2_0
        for layer in self.level3:
            out2 = layer(out2)
        feat = self.b3(torch.cat([out2_0, out2], 1))
        return [self.classifier(feat), None, feat, out2, b2, out1, b1]


def build_student(seed, classes=19, p=2, q=8):
    """Default-initialised ESPNet-C under a fixed seed, BatchNorm running statistics and weights perturbed so that eval mode is
    not trivial, PReLU slopes spread around their 0.25 init (some negative-side gradients then differ per channel)."""
    torch.manual_seed(seed)
    m = ESPNet_Encoder(classes, p, q)
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                c = mod.num_features
                mod.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
                mod.weight.copy_(1.0 + 0.2 * torch.randn(c, generator=g))
                mod.bias.copy_(0.1 * torch.randn(c, generator=g))
            elif isinstance(mod, nn.PReLU):
                mod.weight.copy_(0.25 + 0.1 * torch.randn(mod.weight.numel(), generator=g))
    return m


def resample_teacher(preds_T, size):
    """Decision 1: preds_T[0] and preds_T[-5] bilinear (align_corners=True) onto the student's grid when the shapes differ."""
    if tuple(preds_T[0].shape[2:]) == tuple(size):
        return preds_T
    out = list(preds_T)
    for i in (0, len(out) - 5):
        out[i] = F.interpolate(out[i], size=size, mode="bilinear", align_corners=True)
    return out


def ce_loss(preds, target, ignore_index=255):
    """Decision 2 (CriterionCrossEntropy): CE(up(preds[0])), bilinear align_corners to the label size, mean over valid pixels."""
    up = F.interpolate(preds[0], size=target.shape[1:], mode="bilinear", align_corners=True)
    return F.cross_entropy(up, target, ignore_index=ignore_index)


def size_aware_D(D, logits_hw):
    """The discriminator's 4x4 `last` convolution cut to the map it meets when that map is smaller than 4x4 (2x3 at 45x60 logits),
    as the package's discriminator does; parameters stay registered under `last_conv`."""
    hc, wc = logits_hw
    for _ in range(4):
        hc, wc = (hc - 2) // 2 + 1, (wc - 2) // 2 + 1
    if hc >= 4 and wc >= 4:
        return D
    last = D.last[0]

    class _Head(nn.Module):
        def forward(self, x):
            return F.conv2d(x, last.weight[:, :, :min(4, hc), :min(4, wc)], last.bias)
    D.last_conv = last
    D.last = nn.Sequential(_Head())
    return D


def distill_step(teacher, student, D, images, labels, cfg, gp_alpha=None):
    """networks/kd_model.py:119-164 order with ESPNet-C as the student: forward, G losses and backward, then the discriminator
    phase.  Returns a dict of floats plus preds; gradients stay on the modules' .grad (no optimizer step)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    preds_T = resample_teacher(preds_T, preds_S[0].shape[2:])
    out = {}
    ce = ce_loss(preds_S, labels); out["ce"] = float(ce)
    G = ce
    if cfg.pi:
        t = cfg.lambda_pi * port.pixelwise_loss(preds_S[0], preds_T[0]); out["pi"] = float(t); G = G + t
    if cfg.pa:
        t = port.pairwise_loss(preds_S[2], preds_T[2], cfg.pool_scale); out["pa"] = float(t); G = G + cfg.lambda_pa * t
    if cfg.ho:
        D.train()
        t = cfg.lambda_d * port.adv_loss_g(D(preds_S[0])); out["adv_g"] = float(t); G = G + t
    G.backward(); out["G"] = float(G)
    out["preds_S"], out["preds_T"] = preds_S, preds_T
    if cfg.ho:
        for p in D.parameters():
            p.grad = None
        dT = D(preds_T[0].detach()); dS = D(preds_S[0].detach())
        dl = cfg.lambda_d * port.adv_loss_d(dS, dT, cfg.adv_type)
        if cfg.adv_type == "wgan-gp":
            dl = dl + cfg.lambda_d * port.gradient_penalty(D, preds_S[0], preds_T[0], gp_alpha, cfg.lambda_gp)
        dl.backward(); out["D"] = float(dl)
    return out
