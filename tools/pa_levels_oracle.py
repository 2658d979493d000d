"""Multi-level pair-wise distillation (the reference's kd_model.py:81,137-143, left commented out there): the loop restated over the
oracle ports for every student (float64 when the models and inputs are), the seeded cases, and the generator of
tests/golden/pa_levels.pt.gz.

Level `ind` of `lambda_pa` / `pool_scale` distils preds[-(ind + 1)]: 0 -> x1 (layer1), 1 -> x2, 2 -> x3, 3 -> x4, 4 -> the PSP
features.  A level whose weight is 0 is not computed and logs 0.0.

The generator runs the UNMODIFIED reference on the CPU -- its Res_pspnet student and teacher, and one
CriterionPairWiseforWholeFeatAfterPool(scale=pool_scale[ind], feat_ind=-(ind + 1)) per level -- pins the restatement against it on
the spot, and stores the losses (one Pa term per level), sampled logits and gradient digests:

    SKD_REFERENCE_ROOT=<reference checkout> python -m tools.pa_levels_oracle

TEST INFRASTRUCTURE ONLY.
"""
import gzip
import io
import os
import sys
import time

import torch
import torch.nn.functional as F

from oracle import cases, espnet_port, port

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "pa_levels.pt.gz")

# ResNet18 student, reference goldens.  cfg: port.StepConfig kwargs with list-valued lambda_pa / pool_scale
GOLDEN_CASES = {
    # five levels, mixed scales, x2's weight 0
    "levels5_pi_pa_96x128_b2": dict(batch=2, h=96, w=128, cfg=dict(pi=True, pa=True, ho=False, lambda_pa=[0.5, 0.0, 1.0, 2.0, 0.5],
                                                                    pool_scale=[0.25, 0.5, 0.3, 0.5, 0.125])),
    # a one-entry list distils x1 (preds[-1]), not the PSP features
    "level_x1_pi_pa_96x128_b2": dict(batch=2, h=96, w=128, cfg=dict(pi=True, pa=True, ho=False, lambda_pa=[0.5], pool_scale=[0.25])),
    # the holistic loss beside five levels (65x65 logits: D's 4x4 head fits)
    "levels5_pi_pa_ho_wgangp_512_b1": dict(batch=1, h=512, w=512, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp",
                                                                           lambda_pa=[0.5, 0.5, 0.5, 0.5, 0.5],
                                                                           pool_scale=[0.25, 0.5, 0.125, 0.5, 0.5])),
}

LEVEL_NAMES = ("x1", "x2", "x3", "x4", "psp")


def level_index(ind):
    """preds index of pair-wise level `ind`."""
    return -(ind + 1)


def level_terms(preds_S, preds_T, lambdas, scales):
    """-> (sum_ind lambda[ind] * Pa(preds[-(ind + 1)]) or 0.0, [unweighted term per level, 0.0 where lambda is 0])."""
    total, terms = 0.0, []
    for ind, (lam, scale) in enumerate(zip(lambdas, scales)):
        if lam == 0.0:
            terms.append(0.0)
            continue
        t = port.pairwise_loss(preds_S[level_index(ind)], preds_T[level_index(ind)], scale)
        terms.append(t)
        total = total + lam * t
    return total, terms


def resample_levels(preds_T, preds_S, lambdas):
    """The teacher tensors the losses read -- preds_T[0] and the preds_T[-(ind + 1)] of every level with a non-zero weight --
    each resized (bilinear, align_corners=True) onto the grid of its student counterpart where the grids differ."""
    out = list(preds_T)
    for i in [0] + [len(out) + level_index(ind) for ind, lam in enumerate(lambdas) if lam != 0.0]:
        size = tuple(preds_S[i].shape[2:])
        if tuple(out[i].shape[2:]) != size:
            out[i] = F.interpolate(out[i], size=size, mode="bilinear", align_corners=True)
    return out


def task_loss(kind, preds_S, labels):
    if kind in ("resnet18", "mobilenetv2"):
        return port.dsn_ce_loss(preds_S, labels)
    if kind == "espnet_c":
        return espnet_port.ce_loss(preds_S, labels)
    if kind == "espnet":                                           # logits at the label resolution
        return F.cross_entropy(preds_S[0], labels, ignore_index=255)
    raise ValueError(kind)


def distill_step(kind, teacher, student, D, images, labels, cfg, gp_alpha=None):
    """networks/kd_model.py:119-164 order with the multi-level Pa loop (:137-143): forward, G losses and backward, then the
    discriminator phase.  `cfg.lambda_pa` / `cfg.pool_scale` are lists.  Returns a dict of floats (out["pa"]: one float per level)
    plus preds; gradients stay on the modules' .grad (no optimizer step)."""
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    logits_T = preds_T[0]
    preds_T = resample_levels(preds_T, preds_S, cfg.lambda_pa if cfg.pa else [])
    out = {}
    G = task_loss(kind, preds_S, labels); out["ce"] = float(G)
    if cfg.pi:
        t = cfg.lambda_pi * port.pixelwise_loss(preds_S[0], preds_T[0]); out["pi"] = float(t); G = G + t
    if cfg.pa:
        t, terms = level_terms(preds_S, preds_T, cfg.lambda_pa, cfg.pool_scale)
        out["pa"] = [float(v) for v in terms]; G = G + t
    if kind == "espnet":                                           # the full ESPNet meets D on the teacher's logit grid
        d_in_S, d_in_T = F.interpolate(preds_S[0], size=logits_T.shape[2:], mode="bilinear", align_corners=True), logits_T
    else:
        d_in_S, d_in_T = preds_S[0], preds_T[0]
    if cfg.ho:
        D.train()
        t = cfg.lambda_d * port.adv_loss_g(D(d_in_S)); out["adv_g"] = float(t); G = G + t
    G.backward(); out["G"] = float(G)
    out["preds_S"], out["preds_T"] = preds_S, preds_T
    if cfg.ho:
        for p in D.parameters():
            p.grad = None
        dT = D(d_in_T.detach()); dS = D(d_in_S.detach())
        dl = cfg.lambda_d * port.adv_loss_d(dS, dT, cfg.adv_type)
        if cfg.adv_type == "wgan-gp":
            dl = dl + cfg.lambda_d * port.gradient_penalty(D, d_in_S, d_in_T, gp_alpha, cfg.lambda_gp)
        dl.backward(); out["D"] = float(dl)
    return out


# ----------------------------------------------------------------------------------------------------------- ResNet18 case inputs
def resnet18_case(spec):
    """(teacher, student, D, images, labels, dropout masks, gp alpha) of a golden case, as oracle/make_golden.py seeds them."""
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    masks = cases.dropout_masks(student, spec["batch"], seed=2)
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    return teacher, student, D, images, labels, masks, alpha


def port_step(spec):
    """The restatement on a golden case (fp32, CPU) -> the same record the golden keeps."""
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D, images, labels, masks, alpha = resnet18_case(spec)
    for drop, m in zip(student.dropouts(), masks):
        drop.injected = m
    out = distill_step("resnet18", teacher, student, D if cfg.ho else None, images, labels, cfg, gp_alpha=alpha)
    rec = {k: v for k, v in out.items() if not k.startswith("preds")}
    rec["student_grads"] = cases.grad_digest(student.named_parameters())
    rec["logits_S"] = out["preds_S"][0].detach()[:, :, ::8, ::8].clone()
    if cfg.ho:
        rec["D_grads"] = cases.grad_digest(D.named_parameters())
    return rec


def _ref_step(ref, spec):
    """networks/kd_model.py:119-164 with the multi-level loop of :81,137-143 uncommented, driven by hand with the reference's own
    modules on the CPU (NetModel needs CUDA)."""
    from oracle.make_golden import _cpu_cuda_patch
    C, P = ref.criterion, ref.pspnet
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D, images, labels, masks, alpha = resnet18_case(spec)
    r_student = P.Res_pspnet(P.BasicBlock, [2, 2, 2, 2], num_classes=19)
    r_teacher = P.Res_pspnet(P.Bottleneck, [3, 4, 23, 3], num_classes=19)
    r_student.load_state_dict(student.state_dict(), strict=True)
    r_teacher.load_state_dict(teacher.state_dict(), strict=True)
    for (holder, idx), m in zip(((r_student.pspmodule.bottleneck, 2), (r_student.dsn, 2)), masks):
        cd = port.ChannelDropout(0.1); cd.injected = m                  # identical dropout masks (nn.Dropout2d is torch code)
        holder[idx] = cd
    r_D = None
    if cfg.ho:
        r_D = ref.sagan.Discriminator(1, 19, spec["batch"], 65, 64)
        r_D.load_state_dict(D.state_dict(), strict=True)
    crit_pa = [C.CriterionPairWiseforWholeFeatAfterPool(scale=cfg.pool_scale[ind], feat_ind=-(ind + 1))
               for ind in range(len(cfg.lambda_pa))]                                                        # kd_model.py:81
    r_teacher.eval(); r_student.train()
    with torch.no_grad():
        preds_T = r_teacher(images)
    preds_S = r_student(images)
    out = {}
    G = C.CriterionDSN()(preds_S, labels); out["ce"] = float(G)
    if cfg.pi:
        t = cfg.lambda_pi * C.CriterionPixelWise()(preds_S, preds_T); out["pi"] = float(t); G = G + t
    if cfg.pa:
        pa_G_loss = [0.0] * len(cfg.lambda_pa)
        for ind in range(len(cfg.lambda_pa)):                                                                # kd_model.py:137-143
            if cfg.lambda_pa[ind] != 0.0:
                temp1 = crit_pa[ind](preds_S, preds_T)
                pa_G_loss[ind] = temp1.item()
                G = G + cfg.lambda_pa[ind] * temp1
            elif cfg.lambda_pa[ind] == 0.0:
                pa_G_loss[ind] = 0.0
        out["pa"] = pa_G_loss
    if cfg.ho:
        r_D.train()
        d_out_S = r_D(preds_S[0])
        t = cfg.lambda_d * C.CriterionAdvForG(cfg.adv_type)(d_out_S, d_out_S); out["adv_g"] = float(t); G = G + t
    G.backward(); out["G"] = float(G)
    out["student_grads"] = cases.grad_digest(r_student.named_parameters())
    out["logits_S"] = preds_S[0].detach()[:, :, ::8, ::8].clone()
    out["logits_T"] = preds_T[0].detach()[:, :, ::8, ::8].clone()
    out["feat_norms_T"] = [float(preds_T[level_index(ind)].norm()) for ind in range(len(LEVEL_NAMES))]
    if cfg.ho:
        for p in r_D.parameters():
            p.grad = None
        dT = r_D(preds_T[0].detach()); dS = r_D(preds_S[0].detach())
        dl = cfg.lambda_d * C.CriterionAdv(cfg.adv_type)(dS, dT)
        if cfg.adv_type == "wgan-gp":
            with _cpu_cuda_patch(alpha):
                dl = dl + cfg.lambda_d * C.CriterionAdditionalGP(r_D, cfg.lambda_gp)(preds_S, preds_T)
        dl.backward(); out["D"] = float(dl)
        out["D_grads"] = cases.grad_digest(r_D.named_parameters())
    return out


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def compare(mine, gold):
    """-> dict of relative errors of the restatement's record against the golden's (losses, Pa per level, gradient norms)."""
    rep = {k: _rel(mine[k], gold[k]) for k in ("ce", "pi", "adv_g", "G", "D") if k in gold}
    rep["pa"] = max((_rel(a, b) if b != 0.0 else abs(a)) for a, b in zip(mine["pa"], gold["pa"]))
    rep["student_grad_norm"] = max(_rel(mine["student_grads"][k]["norm"], v["norm"])
                                   for k, v in gold["student_grads"].items() if v["norm"] > 1e-6)
    return rep


def main():
    from oracle import refshim
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    res = {}
    for name, spec in GOLDEN_CASES.items():
        t0 = time.time()
        gold = _ref_step(ref, spec)
        rep = compare(port_step(spec), gold)
        assert all(v < 2e-4 for k, v in rep.items() if k != "student_grad_norm") and rep["student_grad_norm"] < 5e-3, (name, rep)
        print("pa_levels", name, "pa", gold["pa"], "G", gold["G"], "port", {k: "%.1e" % v for k, v in rep.items()},
              "%.1fs" % (time.time() - t0))
        res[name] = gold
    buf = io.BytesIO()
    torch.save(res, buf)
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(buf.getvalue())
    print("written", GOLDEN, "torch", torch.__version__)


def load():
    with gzip.open(GOLDEN, "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


if __name__ == "__main__":
    sys.exit(main())
