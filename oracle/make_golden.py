"""Generate tests/golden/*.pt by running the UNMODIFIED reference Python (the checkout named by SKD_REFERENCE_ROOT, CPU) on the
seeded cases of oracle/cases.py, and pin oracle/port.py against it on the spot.

SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden
TEST INFRASTRUCTURE ONLY.
"""
import contextlib
import os
import sys
import time

import torch

from . import cases, port, refshim

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


@contextlib.contextmanager
def _cpu_cuda_patch(alpha=None):
    """utils/criterion.py:104,109 hard-code .cuda(); on CPU make it the identity and inject torch.rand."""
    orig_cuda, orig_rand = torch.Tensor.cuda, torch.rand
    torch.Tensor.cuda = lambda self, *a, **k: self
    if alpha is not None:
        torch.rand = lambda *a, **k: alpha.clone()
    try:
        yield
    finally:
        torch.Tensor.cuda, torch.rand = orig_cuda, orig_rand


def _rel(a, b):
    a, b = float(a), float(b)
    return abs(a - b) / max(abs(b), 1e-12)


def criterion_goldens(ref):
    out = {}
    for name, n, cs, ct, h, w, scale, (lh, lw) in cases.CRITERION_CASES:
        S, T = cases.criterion_inputs(n, cs, ct, 19, h, w, seed=len(name) * 7 + n)
        g = cases.seeded(5 + n)
        labels = torch.randint(0, 19, (n, lh, lw), generator=g)
        labels[torch.rand(n, lh, lw, generator=g) < 0.05] = 255
        rec = {}
        for t in S[:3]:
            t.requires_grad_(True)
        # --- reference
        pi = ref.criterion.CriterionPixelWise()(S, T)
        pa = ref.criterion.CriterionPairWiseforWholeFeatAfterPool(scale=scale, feat_ind=-5)(S, T)
        ce = ref.criterion.CriterionDSN()(S, labels)
        gi = torch.autograd.grad(pi, S[0], retain_graph=True)[0]
        ga = torch.autograd.grad(pa, S[2], retain_graph=True)[0]
        gc0, gc1 = torch.autograd.grad(ce, [S[0], S[1]])
        rec.update(pi=pi.detach(), pa=pa.detach(), ce=ce.detach(), d_pi=gi, d_pa=ga, d_ce0=gc0, d_ce1=gc1)
        # --- port, pinned now
        p_pi = port.pixelwise_loss(S[0], T[0]); p_pa = port.pairwise_loss(S[2], T[2], scale)
        p_ce = port.dsn_ce_loss(S, labels)
        assert _rel(p_pi, pi) < 1e-6 and _rel(p_pa, pa) < 1e-5 and _rel(p_ce, ce) < 1e-6, (name, p_pi, pi, p_pa, pa)
        assert torch.allclose(torch.autograd.grad(p_pa, S[2])[0], ga, rtol=1e-4, atol=1e-9)
        out[name] = rec
        print("criterion", name, float(pi), float(pa), float(ce))
    return out


def adv_goldens(ref):
    out = {}
    g = cases.seeded(11)
    dS = [torch.randn(4, 1, 1, 5, generator=g)]; dT = [torch.randn(4, 1, 1, 5, generator=g)]
    for adv in ("wgan-gp", "hinge"):
        out[adv] = dict(d=ref.criterion.CriterionAdv(adv)(dS, dT), g=ref.criterion.CriterionAdvForG(adv)(dS, dS))
        assert _rel(port.adv_loss_d(dS, dT, adv), out[adv]["d"]) < 1e-6
        assert _rel(port.adv_loss_g(dS), out[adv]["g"]) < 1e-6
    out["dS"], out["dT"] = dS[0], dT[0]
    return out


def discriminator_golden(ref):
    """D forward x3 (u,v advance), hinge + wgan-gp D losses and gradients on random logits (2,19,65,65)."""
    torch.manual_seed(3)
    Dp = port.Discriminator(1, 19, 64)
    with torch.no_grad():
        Dp.attn1.gamma.fill_(0.3); Dp.attn2.gamma.fill_(-0.2)     # gamma=0 would hide the attention path
    Dr = ref.sagan.Discriminator(1, 19, 2, 65, 64)
    missing = Dr.load_state_dict(Dp.state_dict(), strict=True)
    g = cases.seeded(4)
    xs = torch.randn(2, 19, 65, 65, generator=g) * 3
    xt = torch.randn(2, 19, 65, 65, generator=g) * 3
    alpha = torch.rand(2, 1, 1, 1, generator=g)
    rec = dict(alpha=alpha)
    for tag, D in (("ref", Dr), ("port", Dp)):
        D.train()
        o_s = D(xs); o_t = D(xt)
        if tag == "ref":
            adv = ref.criterion.CriterionAdv("wgan-gp")(o_s, o_t)
            with _cpu_cuda_patch(alpha):
                gp = ref.criterion.CriterionAdditionalGP(D, 10.0)([xs], [xt])
        else:
            adv = port.adv_loss_d(o_s, o_t, "wgan-gp")
            gp = port.gradient_penalty(D, xs, xt, alpha, 10.0)
        (adv + gp).backward()
        rec[tag] = dict(out_s=o_s[0].detach(), p1=o_s[1].detach()[:, :4, :8].clone(), adv=adv.detach(), gp=gp.detach(),
                        grads=cases.grad_digest(D.named_parameters()),
                        u1=D.l1[0].module.weight_u.detach().clone(), bn_rm=D.preprocess_additional.running_mean.clone())
    assert torch.allclose(rec["ref"]["out_s"], rec["port"]["out_s"], rtol=1e-4, atol=1e-5)
    assert _rel(rec["port"]["gp"], rec["ref"]["gp"]) < 1e-4, (rec["port"]["gp"], rec["ref"]["gp"])
    for k, v in rec["ref"]["grads"].items():
        assert _rel(rec["port"]["grads"][k]["norm"], v["norm"]) < 1e-3, k
    print("discriminator adv", float(rec["ref"]["adv"]), "gp", float(rec["ref"]["gp"]))
    return dict(alpha=alpha, **rec["ref"])


def _ref_step(ref, teacher, student, D, images, labels, cfg, alpha):
    """networks/kd_model.py:119-173 driven by hand with the reference's own modules (NetModel needs CUDA)."""
    C = ref.criterion
    teacher.eval(); student.train()
    with torch.no_grad():
        preds_T = teacher(images)
    preds_S = student(images)
    out = {}
    G = C.CriterionDSN()(preds_S, labels); out["ce"] = float(G)
    if cfg.pi:
        t = cfg.lambda_pi * C.CriterionPixelWise()(preds_S, preds_T); out["pi"] = float(t); G = G + t
    if cfg.pa:
        t = C.CriterionPairWiseforWholeFeatAfterPool(scale=cfg.pool_scale, feat_ind=-5)(preds_S, preds_T)
        out["pa"] = float(t); G = G + cfg.lambda_pa * t
    if cfg.ho:
        D.train()
        d_out_S = D(preds_S[0])
        t = cfg.lambda_d * C.CriterionAdvForG(cfg.adv_type)(d_out_S, d_out_S); out["adv_g"] = float(t); G = G + t
    G.backward(); out["G"] = float(G)
    out["student_grads"] = cases.grad_digest(student.named_parameters())
    out["logits_S"] = preds_S[0].detach()[:, :, ::8, ::8].clone()
    out["logits_T"] = preds_T[0].detach()[:, :, ::8, ::8].clone()
    out["feat_T_norm"] = float(preds_T[2].norm())
    if cfg.ho:
        for p in D.parameters():
            p.grad = None
        dT = D(preds_T[0].detach()); dS = D(preds_S[0].detach())
        dl = cfg.lambda_d * C.CriterionAdv(cfg.adv_type)(dS, dT)
        if cfg.adv_type == "wgan-gp":
            with _cpu_cuda_patch(alpha):
                dl = dl + cfg.lambda_d * C.CriterionAdditionalGP(D, cfg.lambda_gp)(preds_S, preds_T)
        dl.backward(); out["D"] = float(dl)
        out["D_grads"] = cases.grad_digest(D.named_parameters())
    return out


def step_goldens(ref, table=None, check_port=True):
    res = {}
    for name, spec in (table or cases.STEP_CASES).items():
        t0 = time.time()
        cfg = port.StepConfig(**spec["cfg"])
        teacher, student, D = cases.build_models(seed=0, with_D=cfg.ho)
        images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
        masks = cases.dropout_masks(student, spec["batch"], seed=2)
        alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
        # reference twins with the same weights
        P = ref.pspnet
        r_student = P.Res_pspnet(P.BasicBlock, [2, 2, 2, 2], num_classes=19)
        r_teacher = P.Res_pspnet(P.Bottleneck, [3, 4, 23, 3], num_classes=19)
        r_student.load_state_dict(student.state_dict(), strict=True)
        r_teacher.load_state_dict(teacher.state_dict(), strict=True)
        r_D = None
        if cfg.ho:
            r_D = ref.sagan.Discriminator(1, 19, spec["batch"], 65, 64)
            r_D.load_state_dict(D.state_dict(), strict=True)
        # inject identical dropout masks on both sides (nn.Dropout2d is torch, not reference, code)
        for drop, m in zip(student.dropouts(), masks):
            drop.injected = m
        for (holder, idx), m in zip(((r_student.pspmodule.bottleneck, 2), (r_student.dsn, 2)), masks):
            cd = port.ChannelDropout(0.1); cd.injected = m
            holder[idx] = cd
        gold = _ref_step(ref, r_teacher, r_student, r_D, images, labels, cfg, alpha)
        if not check_port:
            print("step", name, {k: round(v, 6) for k, v in gold.items() if isinstance(v, float)}, "%.1fs" % (time.time() - t0))
            res[name] = gold
            continue
        mine = port.distill_step(teacher, student, D, images, labels, cfg, gp_alpha=alpha)
        for k in ("ce", "pi", "pa", "adv_g", "G", "D"):
            if k in gold:
                assert _rel(mine[k], gold[k]) < 2e-4, (name, k, mine[k], gold[k])
        mg = cases.grad_digest(student.named_parameters())
        worst = max(_rel(mg[k]["norm"], v["norm"]) for k, v in gold["student_grads"].items() if v["norm"] > 1e-6)
        assert worst < 5e-3, (name, worst)
        print("step", name, {k: round(v, 6) for k, v in gold.items() if isinstance(v, float)},
              "port grad-norm worst rel %.2e" % worst, "%.1fs" % (time.time() - t0))
        res[name] = gold
    return res


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count())
    if "--cfg4" in sys.argv:
        torch.save(step_goldens(ref, cases.CFG4_CASES), os.path.join(GOLDEN_DIR, "steps_cfg4.pt"))
        return
    if "--full" in sys.argv:
        torch.save(step_goldens(ref, cases.FULL_CASES, check_port=False), os.path.join(GOLDEN_DIR, "steps_full.pt"))
        return
    crit = {name: {k: cases.sample_large(v) if torch.is_tensor(v) else v for k, v in g.items()} for name, g in criterion_goldens(ref).items()}
    torch.save(dict(criterion=crit, adv=adv_goldens(ref)), os.path.join(GOLDEN_DIR, "criteria.pt"))
    torch.save(discriminator_golden(ref), os.path.join(GOLDEN_DIR, "discriminator.pt"))
    torch.save(step_goldens(ref), os.path.join(GOLDEN_DIR, "steps.pt"))
    print("golden fixtures written to", GOLDEN_DIR, "torch", torch.__version__)


if __name__ == "__main__":
    sys.exit(main())
