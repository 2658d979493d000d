"""Attention transfer (AT) and MIMIC, the feature-level baselines of the structured-distillation comparison, restated in plain torch
from their definitions (nothing in the reference covers them), and the distillation step with them added after Pa.

  AT    (Zagoruyko & Komodakis):  at(x) = F.normalize(x.pow(2).mean(1).view(N, -1)),  L = mean over N*H*W of (at(S) - at(T))^2
  MIMIC (Li et al.):              L = F.mse_loss(conv1x1(S; weight, bias), T)

Levels follow the pair-wise ones: a scalar weight is one term on preds[-5] (the PSP features), a list puts level `ind` on
preds[-(ind + 1)]; a level with weight 0 is not computed and logs 0.0.  Teacher tensors on another grid than the student's are resized
onto it (bilinear, align_corners=True).  Float64 when the inputs are.  TEST INFRASTRUCTURE ONLY.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import port
from tools import pa_levels_oracle as PL


def level_channels(net, h=64, w=64):
    """Widths of preds[-1] .. preds[-5] of a port network, read off the tensors of an eval-mode forward of one h x w image."""
    was = net.training
    net.eval()
    try:
        with torch.no_grad():
            preds = net(torch.zeros(1, 3, h, w))
    finally:
        net.train(was)
    return tuple(preds[-(ind + 1)].shape[1] for ind in range(5))


def at_map(x):
    n = x.shape[0]
    return F.normalize(x.pow(2).mean(1).view(n, -1))


def at_loss(feat_S, feat_T):
    return (at_map(feat_S) - at_map(feat_T.detach())).pow(2).mean()


def mimic_loss(feat_S, feat_T, adapter):
    return F.mse_loss(adapter(feat_S), feat_T.detach())


def levels(weights):
    """[(feat_ind, weight)] of a scalar (preds[-5]) or a list of weights (level ind on preds[-(ind + 1)]); [] for None."""
    if weights is None:
        return []
    if isinstance(weights, (list, tuple)):
        return [(-(ind + 1), float(w)) for ind, w in enumerate(weights)]
    return [(-5, float(weights))]


def build_adapters(student, teacher, mimic, seed):
    """nn.Conv2d(C_S, C_T, 1) per weighted MIMIC level, C_S / C_T the port networks' widths there, created under torch.manual_seed(seed)
    in level order; keys as NetModel.mimic_adapters."""
    cs, ct = level_channels(student), level_channels(teacher)
    torch.manual_seed(seed)
    return nn.ModuleDict({"level%d" % (-i - 1): nn.Conv2d(cs[-i - 1], ct[-i - 1], 1) for i, w in levels(mimic) if w != 0.0})


def terms(fn, weights, preds_S, preds_T):
    """-> (sum of weight * fn(level ind), the unweighted terms: a list for list weights, else the single one)."""
    total, out = 0.0, []
    for i, w in levels(weights):
        if w == 0.0:
            out.append(0.0)
            continue
        t = fn(i, preds_S[i], preds_T[i])
        out.append(t)
        total = total + w * t
    return total, (out if isinstance(weights, (list, tuple)) else out[0])


def resample(preds_T, preds_S, reads):
    out = list(preds_T)
    for i in reads:
        size = tuple(preds_S[i].shape[2:])
        if tuple(out[i].shape[2:]) != size:
            out[i] = F.interpolate(out[i], size=size, mode="bilinear", align_corners=True)
    return out


def distill_step(kind, teacher, student, D, adapters, images, labels, cfg, at=None, mimic=None, gp_alpha=None):
    """networks/kd_model.py:119-164's step with AT and MIMIC added after Pa (scalar or list lambda_pa): forward, G losses and backward,
    then the discriminator phase.  Returns a dict of floats plus preds; gradients stay on .grad (no optimizer step)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    n = len(preds_T)
    pa_list = isinstance(cfg.lambda_pa, (list, tuple))
    reads = [0]
    if cfg.pa:
        reads += [n - 5] if not pa_list else [n - ind - 1 for ind, w in enumerate(cfg.lambda_pa) if w != 0.0]
    for weights in (at, mimic):
        reads += [n + i for i, w in levels(weights) if w != 0.0 and n + i not in reads]
    preds_T = resample(preds_T, preds_S, reads)
    out = {}
    G = PL.task_loss(kind, preds_S, labels); out["ce"] = float(G)
    if cfg.pi:
        t = cfg.lambda_pi * port.pixelwise_loss(preds_S[0], preds_T[0]); out["pi"] = float(t); G = G + t
    if cfg.pa and pa_list:
        t, pa = PL.level_terms(preds_S, preds_T, cfg.lambda_pa, cfg.pool_scale)
        out["pa"] = [float(v) for v in pa]; G = G + t
    elif cfg.pa:
        t = port.pairwise_loss(preds_S[-5], preds_T[-5], cfg.pool_scale); out["pa"] = float(t); G = G + cfg.lambda_pa * t
    for name, weights, fn in (("at", at, lambda i, s, t: at_loss(s, t)),
                              ("mimic", mimic, lambda i, s, t: mimic_loss(s, t, adapters["level%d" % (-i - 1)]))):
        if weights is not None:
            t, v = terms(fn, weights, preds_S, preds_T)
            out[name] = [float(x) for x in v] if isinstance(v, list) else float(v)
            G = G + t
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
