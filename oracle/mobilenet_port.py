"""The MobileNetV2 student in plain torch -- nn.Conv2d (groups = C for the depthwise layers), nn.BatchNorm2d, nn.ReLU6 in torchvision's
module structure, oracle/port.py's ABN PSP module and DSN head -- and the distillation step with it as the student.  TEST
INFRASTRUCTURE ONLY: the CPU restatement the sm_90a student (structure_knowledge_distillation_b200/networks/mobilenet.py) is checked
against.  The reference has no MobileNetV2, so the architecture is the one the package documents (same attribute names, hence the same
state-dict keys): torchvision's mobilenet_v2 features[0..17], width 1.0, dilated to output stride 8 by CSAIL's MobileNetV2dilated rule,
with the ResNet18 student's head.  torchvision itself is not imported here.

Step decisions: the teacher's tensors are resampled onto the student's grid as for ESPNet (espnet_port.resample_teacher); the task
loss is the DSN cross entropy of the ResNet18 student (port.dsn_ce_loss).
"""
import torch
import torch.nn as nn

from . import espnet_port, port

SETTINGS = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1))


def dilate_of(index):
    return 4 if index >= 14 else (2 if index >= 7 else 1)


class ConvBNReLU(nn.Sequential):
    """torchvision's Conv2dNormActivation: [Conv2d(bias=False), BatchNorm2d, ReLU6]."""

    def __init__(self, cin, cout, k=3, stride=1, groups=1, dilation=1):
        pad = (k - 1) // 2 * dilation
        super().__init__(nn.Conv2d(cin, cout, k, stride, pad, dilation=dilation, groups=groups, bias=False), nn.BatchNorm2d(cout),
                         nn.ReLU6())


class InvertedResidual(nn.Module):
    def __init__(self, cin, cout, stride, t, dilate):
        super().__init__()
        hidden = cin * t
        self.use_res_connect = stride == 1 and cin == cout
        if dilate == 1:
            s, d = stride, 1
        else:
            s, d = 1, (dilate // 2 if stride == 2 else dilate)
        layers = [ConvBNReLU(cin, hidden, k=1)] if t != 1 else []
        layers += [ConvBNReLU(hidden, hidden, 3, s, groups=hidden, dilation=d), nn.Conv2d(hidden, cout, 1, bias=False),
                   nn.BatchNorm2d(cout)]
        self.conv = nn.Sequential(*layers)

    def forward(self, x):
        return x + self.conv(x) if self.use_res_connect else self.conv(x)


def backbone():
    """features[0..17] at output stride 8."""
    feats, cin, i = [ConvBNReLU(3, 32, 3, 2)], 32, 1
    for t, c, n, s in SETTINGS:
        for k in range(n):
            feats.append(InvertedResidual(cin, c, s if k == 0 else 1, t, dilate_of(i)))
            cin, i = c, i + 1
    return nn.Sequential(*feats)


class MobileNetV2Student(nn.Module):
    def __init__(self, classes=19):
        super().__init__()
        self.features = backbone()
        self.pspmodule = port._PSP(320, 128)
        self.head = nn.Conv2d(128, classes, 1, bias=True)
        self.dsn = nn.Sequential(nn.Conv2d(96, 128, 3, 1, 1), port.ABN(128), port.ChannelDropout(0.1),
                                 nn.Conv2d(128, classes, 1, bias=True))

    def dropouts(self):
        return [self.pspmodule.bottleneck[2], self.dsn[2]]

    def forward(self, x):
        keep = {}
        h = x
        for i, f in enumerate(self.features):
            h = f(h)
            keep[i] = h
        x_dsn = self.dsn(keep[13])
        feat = self.pspmodule(keep[17])
        return [self.head(feat), x_dsn, feat, keep[17], keep[13], keep[6], keep[3]]


def dilate_torchvision(model):
    """CSAIL's MobileNetV2dilated `_nostride_dilate` applied to a torchvision mobilenet_v2 in place (features[7..13] dilate 2,
    features[14..17] dilate 4): the twin the oracle's backbone is checked against."""
    for i in range(7, 18):
        dilate = dilate_of(i)
        for m in model.features[i].modules():
            if isinstance(m, nn.Conv2d) and m.kernel_size == (3, 3):
                if m.stride == (2, 2):
                    m.stride = (1, 1)
                    m.dilation = m.padding = (dilate // 2, dilate // 2)
                else:
                    m.dilation = m.padding = (dilate, dilate)
    return model


def build_student(seed, classes=19):
    """Default-initialised student under a fixed seed.  BatchNorm / ABN affine parameters are perturbed, then the running statistics
    are set from one train-mode pass over a seeded batch (momentum 1) and perturbed around it, so that eval mode is neither trivial
    nor degenerate through 17 blocks."""
    torch.manual_seed(seed)
    m = MobileNetV2Student(classes)
    g = torch.Generator().manual_seed(seed + 100)
    norms = [mod for mod in m.modules() if isinstance(mod, (nn.BatchNorm2d, port.ABN))]
    with torch.no_grad():
        for mod in norms:
            c = mod.num_features
            mod.weight.copy_(1.0 + 0.2 * torch.randn(c, generator=g))
            mod.bias.copy_(0.1 * torch.randn(c, generator=g))
        saved = [mod.momentum for mod in norms]
        for mod in norms:
            mod.momentum = 1.0
        for d in m.dropouts():
            d.injected = torch.ones(2, 128)
        m.train()(torch.randn(2, 3, 64, 96, generator=g))
        for d in m.dropouts():
            d.injected = None
        for mod, mo in zip(norms, saved):
            mod.momentum = mo
            c = mod.num_features
            mod.running_mean.add_(0.1 * mod.running_var.sqrt() * torch.randn(c, generator=g))
            mod.running_var.mul_(0.8 + 0.4 * torch.rand(c, generator=g))
            if isinstance(mod, nn.BatchNorm2d):
                mod.num_batches_tracked.zero_()
    return m


def distill_step(teacher, student, D, images, labels, cfg, gp_alpha=None):
    """networks/kd_model.py:119-164 order with MobileNetV2 as the student: the teacher resampled onto the student's grid
    (espnet_port.resample_teacher), the DSN cross entropy, Pi / Pa / Ho as for the other students.  Returns a dict of floats plus
    preds; gradients stay on the modules' .grad (no optimizer step)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    preds_T = espnet_port.resample_teacher(preds_T, preds_S[0].shape[2:])
    out = {}
    ce = port.dsn_ce_loss(preds_S, labels); out["ce"] = float(ce)
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
