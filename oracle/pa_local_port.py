"""Local pair-wise distillation restated in plain torch (float64 when the inputs are), from its definition -- the reference has no local
form -- and the distillation step with it.

Pooling and normalisation are the global term's (oracle/port.py): ceil-mode max pool with window int(H * s) x int(W * s), then
f^ = f / (||f||_2 + 1e-8) with the norm detached, a_ij = f^_i . f^_j on the pooled h x w node grid.  Node i = (y, x) is connected to every
j = (y + t d, x + u d), t, u in -r..r (r = (k - 1) / 2), inside the grid, j = i included, and

    L = sum_n sum_i sum_{j in W(i)} (a^T_ij - a^S_ij)^2 / (N * P),   P = (sum_y c_h(y)) * (sum_x c_w(x)),  c_h(y) = #{t : 0 <= y + t d < h}

With d = 1 and r >= max(h, w) - 1, P = nodes^2 and L is port.pairwise_loss.  The shifted dot products come from slices of the
zero-padded normalised maps: a pair with j outside the grid meets the padding and contributes 0.  TEST INFRASTRUCTURE ONLY.
"""
import torch
import torch.nn.functional as F

from oracle import port
from tools import pa_levels_oracle as PL


def axis_pairs(n, r, d):
    return sum(1 for y in range(n) for t in range(-r, r + 1) if 0 <= y + t * d < n)


def pair_count(h, w, k, d):
    """P: connected ordered pairs per image of an h x w grid."""
    r = (k - 1) // 2
    return axis_pairs(h, r, d) * axis_pairs(w, r, d)


def normalise(feat):
    return feat / ((feat.detach() ** 2).sum(1, keepdim=True).sqrt() + 1e-8)


def local_affinity_loss(ps, pt, k, d):
    """L of the pooled maps ps, pt (N, C_S / C_T, h, w)."""
    return shifted_loss(normalise(ps), normalise(pt.detach()), k, d)


def shifted_loss(fs, ft, k, d):
    """L of the normalised node maps fs, ft (N, C_S / C_T, h, w)."""
    n, _, h, w = fs.shape
    r = (k - 1) // 2
    pad = r * d
    fs, ft = F.pad(fs, (pad,) * 4), F.pad(ft, (pad,) * 4)
    cs, ct = fs[:, :, pad:pad + h, pad:pad + w], ft[:, :, pad:pad + h, pad:pad + w]
    total = 0.0
    for t in range(-r, r + 1):
        for u in range(-r, r + 1):
            y0, x0 = pad + t * d, pad + u * d
            a_s = (cs * fs[:, :, y0:y0 + h, x0:x0 + w]).sum(1)
            a_t = (ct * ft[:, :, y0:y0 + h, x0:x0 + w]).sum(1)
            total = total + ((a_t - a_s) ** 2).sum()
    return total / (n * pair_count(h, w, k, d))


def pairwise_local_loss(feat_S, feat_T, scale, k, d=1):
    """CriterionPairWiseLocal(scale, feat_ind, k, d) on one level's feature maps; the teacher's pooling window sets both."""
    ph, pw = port.pool_patch(feat_T.shape[2], feat_T.shape[3], scale)
    ps = F.max_pool2d(feat_S, (ph, pw), (ph, pw), 0, ceil_mode=True)
    pt = F.max_pool2d(feat_T.detach(), (ph, pw), (ph, pw), 0, ceil_mode=True)
    return local_affinity_loss(ps, pt, k, d)


def pa_term(feat_S, feat_T, scale, window, dilation):
    """The pair-wise term of one level: fully connected when window is None, else local."""
    if window is None:
        return port.pairwise_loss(feat_S, feat_T, scale)
    return pairwise_local_loss(feat_S, feat_T, scale, window, dilation)


def distill_step(kind, teacher, student, D, images, labels, cfg, window=None, dilation=1, gp_alpha=None):
    """networks/kd_model.py:119-164's step with the pair-wise term(s) local where `window` says so: scalars with a scalar
    cfg.lambda_pa (the term on preds[-5]), lists with list cfg.lambda_pa / cfg.pool_scale (level ind on preds[-(ind + 1)], a None window
    fully connected).  Forward, G losses and backward, then the discriminator phase.  Returns a dict of floats plus preds; gradients stay
    on .grad (no optimizer step)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    n = len(preds_T)
    pa_list = isinstance(cfg.lambda_pa, (list, tuple))
    if pa_list:
        preds_T = PL.resample_levels(preds_T, preds_S, cfg.lambda_pa if cfg.pa else [])
    else:
        preds_T = PL.resample_levels(preds_T, preds_S, [])
        if cfg.pa:
            size = tuple(preds_S[n - 5].shape[2:])
            if tuple(preds_T[n - 5].shape[2:]) != size:
                preds_T[n - 5] = F.interpolate(preds_T[n - 5], size=size, mode="bilinear", align_corners=True)
    out = {}
    G = PL.task_loss(kind, preds_S, labels); out["ce"] = float(G)
    if cfg.pi:
        t = cfg.lambda_pi * port.pixelwise_loss(preds_S[0], preds_T[0]); out["pi"] = float(t); G = G + t
    if cfg.pa and pa_list:
        windows = window if isinstance(window, (list, tuple)) else [window] * len(cfg.lambda_pa)
        dilations = dilation if isinstance(dilation, (list, tuple)) else [dilation] * len(cfg.lambda_pa)
        terms = []
        for ind, (lam, scale, k, d) in enumerate(zip(cfg.lambda_pa, cfg.pool_scale, windows, dilations)):
            if lam == 0.0:
                terms.append(0.0)
                continue
            t = pa_term(preds_S[-(ind + 1)], preds_T[-(ind + 1)], scale, k, d)
            terms.append(float(t)); G = G + lam * t
        out["pa"] = terms
    elif cfg.pa:
        t = pa_term(preds_S[-5], preds_T[-5], cfg.pool_scale, window, dilation); out["pa"] = float(t); G = G + cfg.lambda_pa * t
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
