"""Channel-wise distillation (CWD, Shu et al., ICCV 2021) restated in plain torch from its definition (nothing in the reference covers
it), and the distillation step with it added after AT and MIMIC.

  p = softmax over the H*W positions of x / tau, per (image, channel)
  L = tau^2 / (N*C) * sum_{n,c} sum_i pT (log pT - log pS)

log p is log_softmax (max-subtracted), never softmax().log(): that form is -inf wherever pS underflows and makes the loss inf / NaN.
The logit term reads preds[0] (the teacher's logits resized onto the student's grid, as for Pi); feature levels follow the AT / MIMIC
ones (a scalar weight: preds[-5], a list: level `ind` on preds[-(ind + 1)]), each through its own 1x1 adapter from the student's
width to the teacher's.  Float64 when the inputs are.  TEST INFRASTRUCTURE ONLY.
"""
import torch
import torch.nn.functional as F

from oracle import feature_kd_port as FK
from oracle import port
from tools import pa_levels_oracle as PL


def cwd_loss(S, T, tau):
    n, c = S.shape[:2]
    ls = F.log_softmax(S.flatten(2) / tau, -1)
    lt = F.log_softmax(T.detach().flatten(2) / tau, -1)
    return tau * tau * (lt.exp() * (lt - ls)).sum() / (n * c)


def distill_step(kind, teacher, student, D, mimic_adapters, cwd_adapters, images, labels, cfg, at=None, mimic=None, lambda_cwd=3.0,
                 cwd_feat=None, tau=4.0, gp_alpha=None):
    """feature_kd_port.distill_step with CWD after MIMIC: lambda_cwd * CWD(preds[0]) (0: not computed), then the levels of `cwd_feat`
    through `cwd_adapters` (FK.build_adapters' construction, keys as NetModel.cwd_adapters).  out["cwd"] is the logit term alone
    without feature levels, else [logits, level 0, ...].  D sees preds[0] as in feature_kd_port (no full-resolution student with Ho)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    n = len(preds_T)
    pa_list = isinstance(cfg.lambda_pa, (list, tuple))
    reads = [0]
    if cfg.pa:
        reads += [n - 5] if not pa_list else [n - ind - 1 for ind, w in enumerate(cfg.lambda_pa) if w != 0.0]
    for weights in (at, mimic, cwd_feat):
        reads += [n + i for i, w in FK.levels(weights) if w != 0.0 and n + i not in reads]
    preds_T = FK.resample(preds_T, preds_S, reads)
    out = {}
    G = PL.task_loss(kind, preds_S, labels); out["ce"] = float(G)
    if cfg.pi:
        t = cfg.lambda_pi * port.pixelwise_loss(preds_S[0], preds_T[0]); out["pi"] = float(t); G = G + t
    if cfg.pa and pa_list:
        t, pa = PL.level_terms(preds_S, preds_T, cfg.lambda_pa, cfg.pool_scale)
        out["pa"] = [float(v) for v in pa]; G = G + t
    elif cfg.pa:
        t = port.pairwise_loss(preds_S[-5], preds_T[-5], cfg.pool_scale); out["pa"] = float(t); G = G + cfg.lambda_pa * t
    for name, weights, fn in (("at", at, lambda i, s, t: FK.at_loss(s, t)),
                              ("mimic", mimic, lambda i, s, t: FK.mimic_loss(s, t, mimic_adapters["level%d" % (-i - 1)]))):
        if weights is not None:
            t, v = FK.terms(fn, weights, preds_S, preds_T)
            out[name] = [float(x) for x in v] if isinstance(v, list) else float(v)
            G = G + t
    logits = 0.0
    if lambda_cwd != 0.0:
        t = cwd_loss(preds_S[0], preds_T[0], tau); logits = float(t); G = G + lambda_cwd * t
    out["cwd"] = logits
    if cwd_feat is not None:
        t, v = FK.terms(lambda i, s, tt: cwd_loss(cwd_adapters["level%d" % (-i - 1)](s), tt, tau), cwd_feat, preds_S, preds_T)
        out["cwd"] = [logits] + [float(x) for x in (v if isinstance(v, list) else [v])]
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
