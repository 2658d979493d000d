"""TEST INFRASTRUCTURE -- generates tests/golden/disc_preprocess.pt: the discriminator's tanh and rescale input modes
(`preprocess_GAN_mode` 2 and 3, networks/sagan_models.py:147-154) run by the UNMODIFIED reference on the CPU, pinning
oracle/port.py against it on the spot.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_preprocess

Cases:
  * disc_mode2 / disc_mode3: `Discriminator(mode, 19, 2, 65, 64)` on (2, 19, 65, 65) inputs -- D(xs), D(xt), the hinge and wgan-gp D
    losses (CriterionAdv), the penalty (CriterionAdditionalGP, injected alpha; the third call of D), backward of wgan-gp + GP:
    D(xs), the attention map p1 (sampled), losses, GP, u / v of every SN layer after the three calls, gradient digests.
    Inputs: mode 2 takes ordinary logits (3 N(0,1)) with 5 % of xs's entries pushed to |x| in [10, 20] (tanh saturates there);
    mode 3 takes an xs spread uniformly over [0, 255] against ordinary logits as xt.
  * pi_pa_ho_wgangp_512_tanh (mode 2, wgan-gp) / pi_pa_ho_hinge_512_rescale (mode 3, hinge): a full Pi + Pa + Ho distillation step
    at 512 x 512, batch 1, in networks/kd_model.py:119-173 order (make_golden._ref_step), with the seeded models of oracle/cases.py
    and the discriminator built in that mode (its weights are those of cases.build_models' mode-1 D, BatchNorm left out).
"""
import os
import time

import torch

from . import cases, port, refshim
from .make_golden import GOLDEN_DIR, _cpu_cuda_patch, _ref_step, _rel

GOLDEN = os.path.join(GOLDEN_DIR, "disc_preprocess.pt")

STEP_CASES = {
    "pi_pa_ho_wgangp_512_tanh": dict(mode=2, batch=1, h=512, w=512, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
    "pi_pa_ho_hinge_512_rescale": dict(mode=3, batch=1, h=512, w=512, cfg=dict(pi=True, pa=True, ho=True, adv_type="hinge")),
}


def port_D(mode, like):
    """oracle/port.Discriminator in `mode` with the weights of the mode-1 port discriminator `like` (BatchNorm entries dropped)."""
    D = port.Discriminator(mode, 19, 64)
    D.load_state_dict({k: v.clone() for k, v in like.state_dict().items() if not k.startswith("preprocess_additional.")}, strict=True)
    return D


def disc_module(mode):
    """Seeded (D, xs, xt, alpha) of the disc_mode<mode> case; D = oracle/port.Discriminator."""
    torch.manual_seed(3)
    D = port.Discriminator(mode, 19, 64)
    with torch.no_grad():
        D.attn1.gamma.fill_(0.3); D.attn2.gamma.fill_(-0.2)          # gamma = 0 would hide the attention path
    g = cases.seeded(40 + mode)
    xt = torch.randn(2, 19, 65, 65, generator=g) * 3
    if mode == 2:
        xs = torch.randn(2, 19, 65, 65, generator=g) * 3
        far = torch.rand(2, 19, 65, 65, generator=g) < 0.05
        mag = 10 + 10 * torch.rand(2, 19, 65, 65, generator=g)
        xs = torch.where(far, torch.sign(xs) * mag, xs)
    else:
        xs = torch.rand(2, 19, 65, 65, generator=g) * 255
    alpha = torch.rand(2, 1, 1, 1, generator=g)
    return D, xs, xt, alpha


def sn_state(D):
    return {n: (getattr(D, n)[0].module.weight_u.detach().clone(), getattr(D, n)[0].module.weight_v.detach().clone())
            for n in ("l1", "l2", "l3", "l4")}


def disc_golden(ref, mode):
    Dp, xs, xt, alpha = disc_module(mode)
    Dr = ref.sagan.Discriminator(mode, 19, 2, 65, 64)
    Dr.load_state_dict(Dp.state_dict(), strict=True)
    assert sorted(Dr.state_dict()) == sorted(Dp.state_dict())
    rec = {}
    for tag, D in (("ref", Dr), ("port", Dp)):
        D.train()
        o_s = D(xs); o_t = D(xt)
        if tag == "ref":
            hinge = ref.criterion.CriterionAdv("hinge")(o_s, o_t)
            adv = ref.criterion.CriterionAdv("wgan-gp")(o_s, o_t)
            with _cpu_cuda_patch(alpha):
                gp = ref.criterion.CriterionAdditionalGP(D, 10.0)([xs], [xt])
        else:
            hinge = port.adv_loss_d(o_s, o_t, "hinge")
            adv = port.adv_loss_d(o_s, o_t, "wgan-gp")
            gp = port.gradient_penalty(D, xs, xt, alpha, 10.0)
        (adv + gp).backward()
        rec[tag] = dict(out_s=o_s[0].detach(), out_t=o_t[0].detach(), p1=o_s[1].detach()[:, :4, :8].clone(), hinge=hinge.detach(),
                        adv=adv.detach(), gp=gp.detach(), sn=sn_state(D), grads=cases.grad_digest(D.named_parameters()))
    r, p = rec["ref"], rec["port"]
    assert torch.allclose(r["out_s"], p["out_s"], rtol=1e-4, atol=1e-5) and torch.allclose(r["out_t"], p["out_t"], rtol=1e-4, atol=1e-5)
    assert _rel(p["gp"], r["gp"]) < 1e-4 and _rel(p["hinge"], r["hinge"]) < 1e-5, (p["gp"], r["gp"])
    assert sorted(r["grads"]) == sorted(p["grads"])
    for k, v in r["grads"].items():
        assert _rel(p["grads"][k]["norm"], v["norm"]) < 1e-3, k
    print("disc mode", mode, "hinge", float(r["hinge"]), "adv", float(r["adv"]), "gp", float(r["gp"]), flush=True)
    return dict(alpha=alpha, **r)


def step_golden(ref, spec):
    mode, cfg = spec["mode"], port.StepConfig(**spec["cfg"])
    teacher, student, D1 = cases.build_models(seed=0, with_D=True)
    D = port_D(mode, D1)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    masks = cases.dropout_masks(student, spec["batch"], seed=2)
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    P = ref.pspnet
    r_student = P.Res_pspnet(P.BasicBlock, [2, 2, 2, 2], num_classes=19)
    r_teacher = P.Res_pspnet(P.Bottleneck, [3, 4, 23, 3], num_classes=19)
    r_student.load_state_dict(student.state_dict(), strict=True)
    r_teacher.load_state_dict(teacher.state_dict(), strict=True)
    r_D = ref.sagan.Discriminator(mode, 19, spec["batch"], 65, 64)
    r_D.load_state_dict(D.state_dict(), strict=True)
    for drop, m in zip(student.dropouts(), masks):
        drop.injected = m
    for (holder, idx), m in zip(((r_student.pspmodule.bottleneck, 2), (r_student.dsn, 2)), masks):
        cd = port.ChannelDropout(0.1); cd.injected = m
        holder[idx] = cd
    gold = _ref_step(ref, r_teacher, r_student, r_D, images, labels, cfg, alpha)
    mine = port.distill_step(teacher, student, D, images, labels, cfg, gp_alpha=alpha)
    for k in ("ce", "pi", "pa", "adv_g", "G", "D"):
        if k in gold:
            assert _rel(mine[k], gold[k]) < 2e-4, (k, mine[k], gold[k])
    gold["mode"] = mode
    return gold


def main():
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    res = {"disc_mode%d" % m: disc_golden(ref, m) for m in (2, 3)}
    for name, spec in STEP_CASES.items():
        res[name] = step_golden(ref, spec)
        print("step", name, {k: round(v, 6) for k, v in res[name].items() if isinstance(v, float)}, "%.1fs" % (time.time() - t0), flush=True)
    torch.save(res, GOLDEN)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN) // 1024, "KB", "torch", torch.__version__)


if __name__ == "__main__":
    main()
