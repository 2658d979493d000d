"""CPU: the oracle (oracle/port.py) against the golden fixtures produced by the UNMODIFIED reference
(oracle/make_golden.py, run against a checkout of the reference)."""
import os

import pytest
import torch

from oracle import cases, port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gold(name):
    return torch.load(os.path.join(ROOT, "tests", "golden", name), weights_only=False)


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def test_criteria_match_reference():
    gold = _gold("criteria.pt")
    for name, n, cs, ct, h, w, scale, (lh, lw) in cases.CRITERION_CASES:
        S, T = cases.criterion_inputs(n, cs, ct, 19, h, w, seed=len(name) * 7 + n)
        g = cases.seeded(5 + n)
        labels = torch.randint(0, 19, (n, lh, lw), generator=g)
        labels[torch.rand(n, lh, lw, generator=g) < 0.05] = 255
        for t in S[:3]:
            t.requires_grad_(True)
        G = gold["criterion"][name]
        pi = port.pixelwise_loss(S[0], T[0]); pa = port.pairwise_loss(S[2], T[2], scale); ce = port.dsn_ce_loss(S, labels)
        assert _rel(pi, G["pi"]) < 1e-6 and _rel(pa, G["pa"]) < 1e-5 and _rel(ce, G["ce"]) < 1e-6
        (pi + pa + ce).backward()
        assert torch.allclose(*cases.at_stored(S[0].grad, cases.stored_sum(G["d_pi"], G["d_ce0"])), rtol=1e-4, atol=1e-8)
        assert torch.allclose(*cases.at_stored(S[2].grad, G["d_pa"]), rtol=1e-3, atol=1e-9)
    adv = gold["adv"]
    for kind in ("wgan-gp", "hinge"):
        assert _rel(port.adv_loss_d([adv["dS"]], [adv["dT"]], kind), adv[kind]["d"]) < 1e-6
        assert _rel(port.adv_loss_g([adv["dS"]]), adv[kind]["g"]) < 1e-6
    with pytest.raises(ValueError):
        port.adv_loss_d([adv["dS"]], [adv["dT"]], "lsgan")


def test_discriminator_and_gradient_penalty_match_reference():
    gold = _gold("discriminator.pt")
    torch.manual_seed(3)
    D = port.Discriminator(1, 19, 64)
    with torch.no_grad():
        D.attn1.gamma.fill_(0.3); D.attn2.gamma.fill_(-0.2)
    g = cases.seeded(4)
    xs = torch.randn(2, 19, 65, 65, generator=g) * 3
    xt = torch.randn(2, 19, 65, 65, generator=g) * 3
    D.train()
    o_s = D(xs); o_t = D(xt)
    adv = port.adv_loss_d(o_s, o_t, "wgan-gp")
    gp = port.gradient_penalty(D, xs, xt, gold["alpha"], 10.0)
    (adv + gp).backward()
    assert torch.allclose(o_s[0], gold["out_s"], rtol=1e-4, atol=1e-5)
    assert _rel(gp, gold["gp"]) < 1e-4 and _rel(adv, gold["adv"]) < 1e-4
    assert torch.allclose(D.l1[0].module.weight_u, gold["u1"], rtol=1e-5, atol=1e-6)      # u,v advanced 3 times
    for k, v in gold["grads"].items():
        got = dict(D.named_parameters())[k].grad
        assert _rel(got.norm(), v["norm"]) < 1e-3, k


@pytest.mark.parametrize("name", ["cfg1_pi_64", "pi_pa_96x128", "pi_pa_ho_wgangp_512"])
def test_distillation_step_matches_reference(name):
    gold = _gold("steps.pt")[name]
    spec = cases.STEP_CASES[name]
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D = cases.build_models(seed=0, with_D=cfg.ho)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    for drop, m in zip(student.dropouts(), cases.dropout_masks(student, spec["batch"], seed=2)):
        drop.injected = m
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    out = port.distill_step(teacher, student, D, images, labels, cfg, gp_alpha=alpha)
    for k in ("ce", "pi", "pa", "adv_g", "G", "D"):
        if k in gold:
            assert _rel(out[k], gold[k]) < 2e-4, (k, out[k], gold[k])
    mine = cases.grad_digest(student.named_parameters())
    for k, v in gold["student_grads"].items():
        if v["norm"] > 1e-6:
            assert _rel(mine[k]["norm"], v["norm"]) < 5e-3, k


def test_abn_backward_kernel_form_equals_autograd():
    """libs/src/bn.cu:167-232 (y recovered from z, sign-corrected dweight) == autograd through the same forward."""
    g = cases.seeded(9)
    for act in ("none", "leaky_relu", "elu"):
        x = torch.randn(3, 6, 5, 4, generator=g, dtype=torch.float64).requires_grad_(True)
        w = torch.randn(6, generator=g, dtype=torch.float64).requires_grad_(True)
        b = torch.randn(6, generator=g, dtype=torch.float64).requires_grad_(True)
        dz = torch.randn(3, 6, 5, 4, generator=g, dtype=torch.float64)
        rm, rv = torch.zeros(6, dtype=torch.float64), torch.ones(6, dtype=torch.float64)
        z = port._ABNFn.apply(x, w, b, rm, rv, True, 0.1, 1e-5, act, 0.01)
        gx, gw, gb = torch.autograd.grad(z, [x, w, b], dz)
        z2 = port.abn_autograd_equivalent(x, w, b, 1e-5, act, 0.01)
        hx, hw, hb = torch.autograd.grad(z2, [x, w, b], dz)
        assert torch.allclose(gx, hx, rtol=1e-8, atol=1e-10) and torch.allclose(gw, hw, rtol=1e-8) and torch.allclose(gb, hb, rtol=1e-8)
