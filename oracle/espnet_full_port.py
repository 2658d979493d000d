"""The full ESPNet (Mehta et al., ECCV 2018: ESPNet-C plus its decoder, logits at the input resolution) in plain torch --
nn.ConvTranspose2d, nn.BatchNorm2d and the ESPNet-C modules of espnet_port.py -- and the distillation step with it as the student.
TEST INFRASTRUCTURE ONLY: the CPU restatement the sm_90a student (structure_knowledge_distillation_b200/networks/espnet.py, ESPNet)
is checked against.  Same attribute names as the package, hence the same state-dict keys.

Step decisions for a student whose logits are at the input resolution (no reference rule exists for them):
  * CE: the single-head cross entropy on the full-resolution logits; they already have the label size, so there is no upsample;
  * Pi: preds_T[0] is resized (bilinear, align_corners=True) onto the student logits' full-resolution grid, preds_T[-5] onto feat's
    1/8 grid -- each teacher tensor onto the grid of its own student counterpart (for ESPNet-C both are 45x60 at 360x480, which is
    espnet_port.resample_teacher);
  * Pa: unchanged, on feat at 1/8;
  * Ho: the discriminator runs on the teacher's logit grid (46x61 at 360x480).  D(T) sees the teacher logits as they come out, D(S)
    the student logits resized onto that grid (bilinear, align_corners=True), and the gradient penalty interpolates between those
    two.  A full-resolution D would attend over 2 700 (360x480) to 8 192 (512x1024) positions, and the discriminator is built for
    maps of about 65 pixels (imsize_for_adv).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import port
from .espnet_port import BR, C, CBR, DilatedParllelResidualBlockB, ESPNet_Encoder


class ESPNet(nn.Module):
    """ESPNet-C as `encoder` plus the decoder; logits at the input resolution (H, W multiples of 8)."""

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

    def forward(self, x):
        if x.shape[2] % 8 or x.shape[3] % 8:
            raise ValueError("ESPNet needs H and W divisible by 8")
        o = self.encoder(x)
        x3 = self.up_l3(self.br(o[0]))
        y = self.combine_l2_l3(torch.cat([self.level3_C(o[4]), x3], 1))
        y = self.conv(torch.cat([self.up_l2(y), o[6]], 1))
        return [self.classifier(y), None, o[2], o[3], o[4], o[5], o[6]]


def build_student(seed, classes=19, p=2, q=8):
    """Default-initialised full ESPNet under a fixed seed, perturbed as espnet_port.build_student perturbs ESPNet-C: BatchNorm running
    statistics and weights spread so that eval mode is not trivial, PReLU slopes spread around their 0.25 init."""
    torch.manual_seed(seed)
    m = ESPNet(classes, p, q)
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


def teacher_grid(h, w):
    """PSPNet's logit grid for an h x w input: 3x3 / stride-2 stem, ceil-mode 3x3 / stride-2 max pool, stride-2 layer2 (46x61 at
    360x480)."""
    def one(n):
        n = (n - 1) // 2 + 1
        n = -(-(n - 1) // 2) + 1
        return (n - 1) // 2 + 1
    return one(h), one(w)


def resample_teacher_each(preds_T, preds_S):
    """Pi / Pa decision: preds_T[0] and preds_T[-5] each resized (bilinear, align_corners=True) onto the grid of its own student
    counterpart, preds_S[0] and preds_S[-5], where the grids differ."""
    out = list(preds_T)
    for i in (0, len(out) - 5):
        size = tuple(preds_S[i].shape[2:])
        if tuple(out[i].shape[2:]) != size:
            out[i] = F.interpolate(out[i], size=size, mode="bilinear", align_corners=True)
    return out


def distill_step(teacher, student, D, images, labels, cfg, gp_alpha=None):
    """networks/kd_model.py:119-164 order with the full ESPNet as the student and the decisions above: forward, G losses and backward,
    then the discriminator phase (D on the teacher's logit grid; pass a D made size-aware for teacher_grid).  Returns a dict of floats
    plus preds; gradients stay on the modules' .grad (no optimizer step)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    logits_T = preds_T[0]
    preds_T = resample_teacher_each(preds_T, preds_S)
    d_in_S = F.interpolate(preds_S[0], size=logits_T.shape[2:], mode="bilinear", align_corners=True)
    out = {}
    ce = F.cross_entropy(preds_S[0], labels, ignore_index=255); out["ce"] = float(ce)
    G = ce
    if cfg.pi:
        t = cfg.lambda_pi * port.pixelwise_loss(preds_S[0], preds_T[0]); out["pi"] = float(t); G = G + t
    if cfg.pa:
        t = port.pairwise_loss(preds_S[2], preds_T[2], cfg.pool_scale); out["pa"] = float(t); G = G + cfg.lambda_pa * t
    if cfg.ho:
        D.train()
        t = cfg.lambda_d * port.adv_loss_g(D(d_in_S)); out["adv_g"] = float(t); G = G + t
    G.backward(); out["G"] = float(G)
    out["preds_S"], out["preds_T"] = preds_S, preds_T
    if cfg.ho:
        for p in D.parameters():
            p.grad = None
        dT = D(logits_T.detach()); dS = D(d_in_S.detach())
        dl = cfg.lambda_d * port.adv_loss_d(dS, dT, cfg.adv_type)
        if cfg.adv_type == "wgan-gp":
            dl = dl + cfg.lambda_d * port.gradient_penalty(D, d_in_S, logits_T, gp_alpha, cfg.lambda_gp)
        dl.backward(); out["D"] = float(dl)
    return out
