"""Intra-class feature variation distillation (IFVD, Wang et al., ECCV 2020) restated in plain torch from the paper and its authors'
released loss (nothing in the reference covers it), and the distillation step with it added after CWD.

Per feature level, S the student map and T the teacher map (detached), on one h x w grid, K classes:
  lab = F.interpolate(labels[:, None].float(), (h, w), mode="nearest")
  P[n, k] = sum_{lab = k} f / (count + 1e-6), separately for S and T   (IFVD's per-class loop: centre = the prototype of its class)
  cos = F.cosine_similarity(f, centre, dim=1)   (eps 1e-8)
  L = mean over N*h*w of ((cos_S - cos_T) * valid)^2
A pixel whose label is outside [0, K) is its own centre in IFVD's loop (cos(f, f) ~ 1 in both maps); here it is multiplied out, so it
adds exactly 0 to the loss and to the gradient.  The denominator still counts it (nn.MSELoss over the full map).  S gets its gradient
through its cosine and through every prototype it feeds.  Levels follow lambda_at's form (a scalar weight: preds[-5], a list: level
`ind` on preds[-(ind + 1)]).  Float64 when the inputs are.  TEST INFRASTRUCTURE ONLY.
"""
import torch
import torch.nn.functional as F

from oracle import cwd_port
from oracle import feature_kd_port as FK
from oracle import port
from tools import pa_levels_oracle as PL


def labels_nearest(labels, h, w):
    """(N, H, W) labels -> (N, 1, h, w) float labels on the grid (torch's legacy nearest)."""
    return F.interpolate(labels[:, None].float(), (h, w), mode="nearest")


def ifv_loss(feat_S, feat_T, labels, classes_num):
    """IFVD's loss, written as its released per-class loop, with the ignored pixels multiplied out of (cos_S - cos_T)."""
    feat_T = feat_T.detach()
    lab = labels_nearest(labels, *feat_S.shape[2:]).to(feat_S.dtype)
    tar_S, tar_T = lab.expand(feat_S.size()), lab.expand(feat_T.size())
    center_S, center_T = feat_S.clone(), feat_T.clone()
    for i in range(classes_num):
        mask_S = (tar_S == i).to(feat_S.dtype)
        mask_T = (tar_T == i).to(feat_T.dtype)
        center_S = (1 - mask_S) * center_S + mask_S * ((mask_S * feat_S).sum(-1).sum(-1) /
                                                       (mask_S.sum(-1).sum(-1) + 1e-6)).unsqueeze(-1).unsqueeze(-1)
        center_T = (1 - mask_T) * center_T + mask_T * ((mask_T * feat_T).sum(-1).sum(-1) /
                                                       (mask_T.sum(-1).sum(-1) + 1e-6)).unsqueeze(-1).unsqueeze(-1)
    cos_S = F.cosine_similarity(feat_S, center_S, dim=1)
    cos_T = F.cosine_similarity(feat_T, center_T, dim=1)
    valid = ((lab[:, 0] >= 0) & (lab[:, 0] < classes_num)).to(feat_S.dtype)
    return F.mse_loss(cos_S * valid, cos_T * valid)


def ifv_loss_scatter(feat_S, feat_T, labels, classes_num):
    """The same term restated with index_add over (image, class) rows instead of the loop (an independent check of ifv_loss)."""
    feat_T = feat_T.detach()
    n, _, h, w = feat_S.shape
    lab = labels_nearest(labels, h, w)[:, 0].long().reshape(n, h * w)
    valid = (lab >= 0) & (lab < classes_num)
    row = (torch.arange(n)[:, None] * classes_num + lab.clamp(0, classes_num - 1)).reshape(-1)   # (n * h * w,)
    vflat = valid.reshape(-1)

    def cosines(f):
        fl = f.flatten(2).transpose(1, 2).reshape(n * h * w, -1)
        keep = vflat.to(f.dtype)[:, None]
        sums = torch.zeros(n * classes_num, fl.shape[1], dtype=f.dtype).index_add(0, row, fl * keep)
        cnt = torch.zeros(n * classes_num, dtype=f.dtype).index_add(0, row, keep[:, 0])
        proto = sums / (cnt[:, None] + 1e-6)
        return F.cosine_similarity(fl, proto[row], dim=1)

    d = (cosines(feat_S) - cosines(feat_T)) * vflat.to(feat_S.dtype)
    return d.pow(2).sum() / (n * h * w)


def distill_step(kind, teacher, student, D, mimic_adapters, cwd_adapters, images, labels, cfg, at=None, mimic=None, lambda_cwd=0.0,
                 cwd_feat=None, tau=4.0, ifv=None, classes_num=19, gp_alpha=None):
    """cwd_port.distill_step with IFV after CWD: the levels of `ifv` (lambda_at's form; None: off) each weight * ifv_loss on the
    student's grid, the teacher resampled there.  out["ifv"] is the unweighted term, a list for list weights.  CWD terms are computed
    only when asked (lambda_cwd != 0 or cwd_feat)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    n = len(preds_T)
    pa_list = isinstance(cfg.lambda_pa, (list, tuple))
    reads = [0]
    if cfg.pa:
        reads += [n - 5] if not pa_list else [n - ind - 1 for ind, w in enumerate(cfg.lambda_pa) if w != 0.0]
    for weights in (at, mimic, cwd_feat, ifv):
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
    if lambda_cwd != 0.0:
        t = cwd_port.cwd_loss(preds_S[0], preds_T[0], tau); out["cwd"] = float(t); G = G + lambda_cwd * t
    if cwd_feat is not None:
        t, v = FK.terms(lambda i, s, tt: cwd_port.cwd_loss(cwd_adapters["level%d" % (-i - 1)](s), tt, tau), cwd_feat, preds_S, preds_T)
        out["cwd"] = [out.get("cwd", 0.0)] + [float(x) for x in (v if isinstance(v, list) else [v])]
        G = G + t
    if ifv is not None:
        t, v = FK.terms(lambda i, s, tt: ifv_loss(s, tt, labels, classes_num), ifv, preds_S, preds_T)
        out["ifv"] = [float(x) for x in v] if isinstance(v, list) else float(v)
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
