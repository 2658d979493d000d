"""CPU: the discriminator's tanh and rescale input modes (preprocess_GAN_mode 2 / 3, networks/sagan_models.py:147-154).

  * oracle/gp_dual_preprocess.py's "reverse over forward" penalty gradient against torch's double backward of oracle/port.py in float64;
  * oracle/port.py against tests/golden/disc_preprocess.pt, written by the UNMODIFIED reference (oracle/make_golden_preprocess.py);
  * the module surface: parameter list, state-dict keys, optimizer flat buffer and checkpoint loading carry no
    `preprocess_additional.*` entry, as in the reference."""
import copy
import os

import pytest
import torch

from oracle import cases, gp_dual_preprocess, make_golden_preprocess as mgp, port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "disc_preprocess.pt"), weights_only=False)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().flatten(), torch.as_tensor(b).double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("mode", [2, 3])
@pytest.mark.parametrize("shape", [(2, 65, 65), (2, 65, 129)])
def test_dual_pass_equals_double_backward(mode, shape):
    B, H, W = shape
    torch.manual_seed(3)
    D = port.Discriminator(mode, 19, 64).double()
    with torch.no_grad():
        D.attn1.gamma.fill_(0.3); D.attn2.gamma.fill_(-0.2)          # gamma = 0 would hide the attention path
    D.train()
    D2 = copy.deepcopy(D)
    g = torch.Generator().manual_seed(H + mode)
    if mode == 2:                                                    # ordinary logits, some saturating tanh
        xs = torch.randn(B, 19, H, W, generator=g, dtype=torch.float64) * 3
        xs[torch.rand(B, 19, H, W, generator=g) < 0.05] *= 5
    else:                                                            # values over [0, 255]
        xs = torch.rand(B, 19, H, W, generator=g, dtype=torch.float64) * 255
    xt = torch.randn(B, 19, H, W, generator=g, dtype=torch.float64) * 3
    alpha = torch.rand(B, 1, 1, 1, generator=g, dtype=torch.float64)
    gp = port.gradient_penalty(D, xs, xt, alpha, 10.0)
    gp.backward()
    gp2, grads = gp_dual_preprocess.gp_and_param_grads(D2, alpha * xt + (1 - alpha) * xs, 10.0)
    assert abs(float(gp.detach()) - float(gp2)) < 1e-8 * abs(float(gp2))
    assert torch.allclose(D.l1[0].module.weight_u, D2.l1[0].module.weight_u)
    # every trainable parameter is covered (last.0.bias, which the penalty does not reach, as zeros) and nothing else
    assert set(grads) == {n for n, p in D.named_parameters() if p.requires_grad}
    for name, p in D.named_parameters():
        if p.grad is None:
            continue
        scale = float(p.grad.norm())
        assert float((p.grad - grads[name]).norm()) <= 1e-7 * scale + 1e-15, name


@pytest.mark.parametrize("mode", [2, 3])
def test_port_matches_reference_golden(gold, mode):
    """Same sequence as the generator: D(xs), D(xt), hinge / wgan-gp losses, GP (third call), backward of wgan-gp + GP."""
    r = gold["disc_mode%d" % mode]
    D, xs, xt, alpha = mgp.disc_module(mode)
    assert torch.equal(alpha, r["alpha"])
    D.train()
    o_s, o_t = D(xs), D(xt)
    hinge, adv = port.adv_loss_d(o_s, o_t, "hinge"), port.adv_loss_d(o_s, o_t, "wgan-gp")
    gp = port.gradient_penalty(D, xs, xt, alpha, 10.0)
    (adv + gp).backward()
    assert _rel(o_s[0].detach(), r["out_s"]) < 1e-5 and _rel(o_t[0].detach(), r["out_t"]) < 1e-5
    assert _rel(o_s[1].detach()[:, :4, :8], r["p1"]) < 1e-5
    assert _rel(hinge.detach(), r["hinge"]) < 1e-5 and _rel(gp.detach(), r["gp"]) < 1e-4
    assert abs(float(adv) - float(r["adv"])) < 1e-5 * float(r["out_s"].abs().mean())
    for name, (u, v) in mgp.sn_state(D).items():
        assert _rel(u, r["sn"][name][0]) < 1e-5 and _rel(v, r["sn"][name][1]) < 1e-5, name
    mine = cases.grad_digest(D.named_parameters())
    assert set(mine) == set(r["grads"])
    for k, v in r["grads"].items():
        assert abs(mine[k]["norm"] - v["norm"]) <= 1e-3 * v["norm"] + 1e-7, k


@pytest.mark.parametrize("mode", [2, 3])
def test_module_surface_matches_reference(gold, mode, tmp_path):
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.optim import FlatSGD
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    from structure_knowledge_distillation_b200.utils.utils import load_D_model
    D = Discriminator(mode, 19, 2, 65, 64)
    ref_params = set(gold["disc_mode%d" % mode]["grads"])           # the reference's trainable parameters (all receive a gradient)
    assert set(D.grad_names) == ref_params
    assert not any(k.startswith("preprocess_additional") for k in D.state_dict())
    assert set(D.state_dict()) == set(port.Discriminator(mode, 19, 64).state_dict())
    D.train(); D.eval()                                              # no parameters or buffers for train() / eval() to switch
    x = torch.linspace(-300, 300, 1001)
    ref_map = torch.tanh(x) if mode == 2 else 2 * (x / 255 - 0.5)
    assert torch.equal(D.preprocess_additional(x), ref_map)          # the reference's module / lambda, kept as the attribute
    # the discriminator optimizer's flat buffer holds only the SN, attention and last-conv parameters
    opt = FlatSGD([p for p in D.parameters() if p.requires_grad], 4e-4, momentum=0.9, weight_decay=5e-4)
    assert opt.flat_p.numel() == sum((p.numel() + 3) // 4 * 4 for n, p in D.named_parameters() if n in ref_params)
    # checkpoint round trip through load_D_model (utils/utils.py:129-151), keys saved from an nn.DataParallel wrapper
    src = Discriminator(mode, 19, 2, 65, 64)
    with torch.no_grad():
        for p in src.parameters():
            p.add_(0.5)
    torch.save(dict(epoch=3, best_mean_IU=0.25, state_dict={"module." + k: v for k, v in src.state_dict().items()}),
               str(tmp_path / "model_best.pth.tar"))
    args = make_args(preprocess_GAN_mode=mode, D_resume=True, D_ckpt_path=str(tmp_path))
    dst = Discriminator(mode, 19, 2, 65, 64)
    assert load_D_model(args, dst, False) == "resume"
    assert args.start_epoch == 3 and args.best_mean_IU == 0.25
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v), k
