"""Attention transfer (AT) and MIMIC on the H100: the csrc/feature_kd.cu kernels against float64 autograd, the MIMIC adapter's
convolution launches bit for bit on exact integer data, NetModel steps against tests/golden/feature_kd.pt.gz (oracle/feature_kd_port.py),
CUDA-graph replay, repeatability, the training-state file and resume, two NCCL ranks, and the defaults launching none of it."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _relf(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _nhwc(n, c, h, w, gen, pitch=None, scale=1.0):
    """(N, C, H, W) view of a random NHWC buffer, a channel slice of a `pitch`-wide one when given (as the teacher's x4 is)."""
    p = pitch or c
    buf = torch.randn(n, h, w, p, generator=gen, device="cuda") * scale
    return buf.permute(0, 3, 1, 2)[:, p - c:] if pitch else buf.permute(0, 3, 1, 2)


def _at_ref(S, T):
    from oracle import feature_kd_port as P
    sd = S.detach().double().contiguous().requires_grad_(True)
    loss = P.at_loss(sd, T.double())
    (g,) = torch.autograd.grad(loss, sd)
    return loss, g


# (N, C_S, C_T, H, W, student pitch, teacher pitch)
AT_CASES = [
    (1, 32, 128, 13, 17, None, None),
    (2, 128, 512, 33, 65, None, None),
    (3, 512, 2048, 17, 31, None, 4096),          # ResNet18 x4 against the teacher's x4, a slice of the PSP concat buffer
    (8, 19, 256, 23, 29, 20, None),              # ESPNet's b1: 19 of 20 channels, scalar path
    (5, 131, 1022, 11, 9, 132, 1025),            # ESPNet's b2 width; the teacher 3 floats into a 1025-wide buffer: misaligned, scalar path
    (4, 2048, 32, 7, 15, None, None),
]


@pytest.mark.parametrize("case", AT_CASES, ids=lambda c: "N%d_C%d-%d_%dx%d" % c[:5])
def test_at_matches_float64(case):
    """Loss and student gradient against autograd through F.normalize in float64.  Bound: the channel mean of squares and the loss are
    fp32 sums (up to 2048 terms per pixel, fp32 FMAs, so at most C * 2^-24 = 1.2e-4 relative, typically sqrt(C) * 2^-24); norms and the
    loss's final sum run in double.  Independent S and T keep the loss free of cancellation."""
    from structure_knowledge_distillation_b200 import functions as Fn
    n, cs, ct, h, w, ps, pt = case
    gen = torch.Generator(device="cuda").manual_seed(sum(case[:5]))
    S, T = _nhwc(n, cs, h, w, gen, ps), _nhwc(n, ct, h, w, gen, pt)
    Sg = S.detach().requires_grad_(True)
    loss = Fn.AttentionTransferLoss.apply(Sg, T)
    (g,) = torch.autograd.grad(loss * 3.0, Sg)
    ref, gref = _at_ref(S, T)
    e_loss, e_grad = _relf(loss, ref), _rel(g.double(), 3.0 * gref)
    print("\nPARITY at", case, "loss %.2e grad %.2e" % (e_loss, e_grad))
    assert e_loss < 2e-5 and e_grad < 1e-4, (e_loss, e_grad)
    if ps:
        assert g.stride() == S.stride()                           # the gradient keeps the student's pitched layout


def test_at_clamped_and_zero_maps():
    """F.normalize's clamp: a student map whose ||q|| is below 1e-12 (values ~1e-8, so q ~ 1e-16) is divided by 1e-12 and its gradient
    is h / 1e-12; an all-zero map has q = 0 and a zero gradient; the loss matches float64 in both."""
    from structure_knowledge_distillation_b200 import functions as Fn
    gen = torch.Generator(device="cuda").manual_seed(5)
    for scale in (1e-8, 0.0):
        S = _nhwc(2, 64, 9, 11, gen, scale=scale)
        T = _nhwc(2, 256, 9, 11, gen)
        Sg = S.detach().requires_grad_(True)
        loss = Fn.AttentionTransferLoss.apply(Sg, T)
        (g,) = torch.autograd.grad(loss, Sg)
        ref, gref = _at_ref(S, T)
        print("\nPARITY at clamp scale", scale, float(loss), float(ref), float(g.abs().max()), float(gref.abs().max()))
        assert _relf(loss, ref) < 1e-5
        if scale:
            assert float(S.double().pow(2).mean(1).flatten(1).norm(dim=1).max()) < 1e-12
            assert _rel(g.double(), gref) < 1e-4
        else:
            assert torch.count_nonzero(g) == 0 and torch.count_nonzero(gref) == 0


# (N, C, H, W, adapter-output pitch, teacher pitch)
MSE_CASES = [(1, 32, 13, 17, None, None), (2, 128, 33, 65, None, None), (3, 2048, 17, 31, None, 4096), (8, 19, 23, 29, 20, 20),
             (4, 512, 7, 15, None, 516), (2, 64, 9, 13, None, 67)]      # last: teacher 3 floats into a 67-wide buffer, scalar path


@pytest.mark.parametrize("case", MSE_CASES, ids=lambda c: "N%d_C%d_%dx%d" % c[:4])
def test_mse_matches_float64(case):
    """F.mse_loss and its gradient in float64.  Bound: squared differences summed in double per thread, one fp32 rounding of each
    difference and square: 2^-23 relative."""
    from structure_knowledge_distillation_b200 import functions as Fn
    n, c, h, w, pr, pt = case
    gen = torch.Generator(device="cuda").manual_seed(sum(case[:4]))
    R, T = _nhwc(n, c, h, w, gen, pr), _nhwc(n, c, h, w, gen, pt)
    Rg = R.detach().requires_grad_(True)
    loss = Fn.MseLoss.apply(Rg, T)
    (g,) = torch.autograd.grad(loss * 0.5, Rg)
    rd = R.detach().double().requires_grad_(True)
    ref = torch.nn.functional.mse_loss(rd, T.double())
    (gref,) = torch.autograd.grad(ref * 0.5, rd)
    e_loss, e_grad = _relf(loss, ref), _rel(g.double(), gref)
    print("\nPARITY mse", case, "loss %.2e grad %.2e" % (e_loss, e_grad))
    assert e_loss < 1e-6 and e_grad < 1e-6, (e_loss, e_grad)


def _resnet18(batch, h, w, cfg, **extra):
    """NetModel with the ResNet18 student on the seeded weights, dropout masks, adapters and batch of the golden cases."""
    from oracle import cases, feature_kd_port, make_golden_feature_kd as G, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**cfg)
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    m = NetModel(make_args(batch_size=batch, pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, **extra))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    if m.mimic:
        m.mimic_adapters.load_state_dict(feature_kd_port.build_adapters(student, teacher, extra["lambda_mimic"], G.ADAPTER_SEED).state_dict())
    for drop, mk in zip(m.student.dropouts(), cases.dropout_masks(student, batch, seed=2)):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    return m


def test_real_x4_levels_match_float64():
    """AT and MIMIC on the features of a real forward (ResNet18, 256x256, batch 2) at x4: the teacher's x4 is its pitched slice of the
    PSP concat buffer, the adapter 512 -> 2048.  Adapter output against F.conv2d in float64 sets the TF32 scale of the bound."""
    from oracle import feature_kd_port as P
    m = _resnet18(2, 256, 256, dict(pi=False, pa=False, ho=False), at=True, lambda_at=[0.0, 0.0, 0.0, 1.0], mimic=True,
                  lambda_mimic=[0.0, 0.0, 0.0, 1.0])
    m.forward()
    fS, fT = m.preds_S[-4].detach(), m.preds_T[-4]
    assert fT.stride(3) == 2048 + 4 * 512 and fT.stride(1) == 1
    rep = {}
    Sg = fS.clone().requires_grad_(True)
    loss = m.criterion_at[3]([None] * 3 + [Sg] + [None] * 3, m.preds_T)
    (g,) = torch.autograd.grad(loss, Sg)
    ref, gref = _at_ref(fS, fT)
    rep["at"], rep["at_grad"] = _relf(loss, ref), _rel(g.double(), gref)
    ad = m.mimic_adapters["level3"]
    Sg = fS.clone().requires_grad_(True)
    loss = m.criterion_mimic[3]([None] * 3 + [Sg] + [None] * 3, m.preds_T)
    (g,) = torch.autograd.grad(loss, Sg)
    sd = fS.double().requires_grad_(True)
    conv = torch.nn.Conv2d(512, 2048, 1).cuda().double()
    conv.weight.data.copy_(ad.weight.double()); conv.bias.data.copy_(ad.bias.double())
    ref = P.mimic_loss(sd, fT.double(), conv)
    (gref,) = torch.autograd.grad(ref, sd)
    rep["mimic"], rep["mimic_grad"] = _relf(loss, ref), _rel(g.double(), gref)
    print("\nPARITY feature_kd x4", rep)
    assert rep["at"] < 2e-5 and rep["at_grad"] < 1e-4
    assert rep["mimic"] < 2e-3 and rep["mimic_grad"] < 1e-2          # TF32 operands of the 512-deep adapter (test_kernels_gpu.py's scale)


# -------------------------------------------------------------------------------------------- the adapter's launches on exact data
LIMIT = 1 << 22                 # largest sum of |terms| of one output element: every fp32 product and sum is exact in any order


@pytest.mark.parametrize("cin, cout, n, h, w", [(128, 512, 2, 65, 65), (512, 2048, 1, 33, 41), (256, 1024, 2, 12, 16),
                                                (19, 256, 1, 45, 60), (24, 256, 2, 32, 64)])
def test_adapter_launches_exact(cin, cout, n, h, w):
    """The MIMIC adapter's forward (bias in the epilogue), data gradient, weight gradient and bias column sum, bit for bit equal to
    float64 on small integers (tests/test_conv_exact_gpu.py's rule: every |sum of terms| <= 2^22, TF32-exact operands)."""
    from structure_knowledge_distillation_b200 import functions as Fn
    from structure_knowledge_distillation_b200.networks.pspnet_combine import Conv2d
    gen = torch.Generator(device="cuda").manual_seed(cin + cout + h)
    ad = Conv2d(cin, cout, 1, bias=True).cuda()
    P = n * h * w
    a_x = max(1, min(math.isqrt(LIMIT // (4 * cin)), 1 << 10))
    x = torch.randint(-a_x, a_x + 1, (n, h, w, cin), generator=gen, device="cuda").float().permute(0, 3, 1, 2)
    with torch.no_grad():
        ad.weight.copy_(torch.randint(-a_x, a_x + 1, (cout, cin, 1, 1), generator=gen, device="cuda").float())
        ad.bias.copy_(torch.randint(-1024, 1025, (cout,), generator=gen, device="cuda").float())
    a_dy = max(1, min(LIMIT // max(P * a_x, cout * a_x), 1 << 10))
    dy = torch.randint(-a_dy, a_dy + 1, (n, h, w, cout), generator=gen, device="cuda").float().permute(0, 3, 1, 2)
    # keep the weight-gradient sums (P terms of |x| * |dy|) inside the exact range
    bound = float((x.abs().reshape(-1, cin).double().t() @ dy.abs().permute(0, 2, 3, 1).reshape(-1, cout).double()).max())
    bound = max(bound, float((dy.abs().permute(0, 2, 3, 1).reshape(-1, cout).double() @ ad.weight.abs().reshape(cout, cin).double()).max()))
    assert bound <= LIMIT and float((x.abs().permute(0, 2, 3, 1).reshape(-1, cin).double() @ ad.weight.abs().reshape(cout, cin).double().t()).max()) <= LIMIT
    xg = x.detach().requires_grad_(True)
    y = ad(xg)
    y.backward(dy)
    xd, wd, bd = x.double(), ad.weight.detach().double(), ad.bias.detach().double()
    yref = torch.nn.functional.conv2d(xd, wd, bd)
    dxref = torch.nn.functional.conv_transpose2d(dy.double(), wd)
    dwref = torch.einsum("nohw,nihw->oi", dy.double(), xd).reshape(cout, cin, 1, 1)
    dbref = dy.double().sum((0, 2, 3))
    assert torch.equal(y.double(), yref)
    assert torch.equal(xg.grad.double(), dxref)
    assert torch.equal(ad.weight.grad.double(), dwref)
    assert torch.equal(ad.bias.grad.double(), dbref)


# -------------------------------------------------------------------------------------------- NetModel steps against the golden
def _case_model(spec):
    from oracle import cases, espnet_port, feature_kd_port, make_golden_feature_kd as G, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**spec["cfg"])
    teacher, student, D, adapters, images, labels, masks, alpha = G.case_inputs(spec)
    m = NetModel(make_args(batch_size=spec["batch"], pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, student=spec["kind"],
                           at=True, lambda_at=spec["at"], mimic=True, lambda_mimic=spec["mimic"]))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    m.mimic_adapters.load_state_dict(adapters.state_dict())
    for drop, mk in zip(m.student.dropouts(), masks):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = alpha.cuda()
    m.set_input((images, labels, None, None))
    return m, c


def _samples(named, digest):
    """(mine, gold) rows of sampled values normalised by the golden's norm, and the worst relative norm error."""
    worst, mine_s, gold_s = 0.0, [], []
    for name, v in named:
        gd = digest.get(name)
        if gd is None or gd["norm"] < 1e-6:
            continue
        a = v.detach().flatten().double()
        worst = max(worst, abs(float(a.norm()) - gd["norm"]) / gd["norm"])
        mine_s.append(a[gd["idx"].to(a.device)].cpu() / gd["norm"]); gold_s.append(gd["samples"].double() / gd["norm"])
    return torch.cat(mine_s), torch.cat(gold_s), worst


@pytest.mark.parametrize("name", ["r18_pi_pa_ho_at_mimic_psp_512_b1", "r18_at5_mimic_x3_96x128_b2", "espnet_c_at5_mimic_psp_360x480_b1"])
def test_step_matches_golden(name):
    """Losses, logits, sampled student and adapter gradients and the parameters after one SGD step against the fp32 CPU restatement.
    Bounds are tests/test_pa_levels_gpu.py's: the random-init student runs TF32 convolutions whose rounding batch-statistic BN amplifies,
    so gradients agree in direction and norm, not to fp32.  The task and Pi losses agree to 1e-3, Pa and MIMIC (read from the student's
    features) to 5e-3, AT (a difference of normalised maps of those features) to 1e-2; the adapters' gradients, one 1x1 layer from the
    loss, to 0.1."""
    from oracle import make_golden_feature_kd as G
    gold = G.load()[name]
    m, cfg = _case_model(G.GOLDEN_CASES[name])
    p0 = {k: p.detach().clone() for k, p in list(m.student.named_parameters()) + list(m.mimic_adapters.named_parameters())}
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    rep = dict(ce=_relf(m.mc_G_loss, gold["ce"]), G=_relf(m.G_loss, gold["G"]))
    if cfg.pi:
        rep["pi"] = _relf(m.pi_G_loss, gold["pi"])
    if cfg.pa:
        rep["pa"] = _relf(m.pa_G_loss, gold["pa"])
    for term in ("at", "mimic"):
        mine, ref = getattr(m, term + "_G_loss"), gold[term]
        mine, ref = (mine, ref) if isinstance(ref, list) else ([mine], [ref])
        assert len(mine) == len(ref)
        for ind, (a, b) in enumerate(zip(mine, ref)):
            if b == 0.0:
                assert a == 0.0 and isinstance(a, float)
            else:
                rep["%s%d" % (term, ind)] = _relf(a, b)
    rep["logits_S"] = _rel(m.preds_S[0][:, :, ::8, ::8].float().cpu(), gold["logits_S"])
    for what, named, digest in (("student", m.student.named_parameters(), gold["student_grads"]),
                                ("adapter", m.mimic_adapters.named_parameters(), gold["adapter_grads"])):
        sm, sg, worst = _samples([(k, p.grad) for k, p in named], digest)
        rep[what + "_grad_norm"], rep[what + "_grad_l2"] = worst, float((sm - sg).norm() / sg.norm())
        rep[what + "_grad_cos"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    m.G_solver.step()
    for what, named, update in (("student", m.student.named_parameters(), gold["student_update"]),
                                ("adapter", m.mimic_adapters.named_parameters(), gold["adapter_update"])):
        digest = gold[what + "_grads"]
        mine, ref = [], []
        for k, p in named:
            if k in update and digest[k]["norm"] >= 1e-6:
                d = (p.detach() - p0[k]).flatten().double()[digest[k]["idx"].to(p.device)].cpu()
                mine.append(d / digest[k]["norm"]); ref.append(update[k].double() / digest[k]["norm"])
        a, b = torch.cat(mine), torch.cat(ref)
        rep[what + "_update_l2"] = float((a - b).norm() / b.norm())
    print("\nPARITY feature_kd step", name, {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        if k in ("ce", "pi", "G"):
            assert v < 1e-3, (k, v)
        elif k == "pa" or k.startswith("mimic"):
            assert v < 5e-3, (k, v)
        elif k.startswith("at"):
            assert v < 1e-2, (k, v)
    assert rep["logits_S"] < 3e-2
    assert rep["student_grad_norm"] < 0.6 and rep["student_grad_l2"] < 0.35 and rep["student_grad_cos"] > 0.93
    assert rep["student_update_l2"] < 0.35
    assert rep["adapter_grad_norm"] < 0.1 and rep["adapter_grad_l2"] < 0.1 and rep["adapter_grad_cos"] > 0.99
    assert rep["adapter_update_l2"] < 0.1


@pytest.mark.parametrize("kind", ["mobilenetv2", "espnet"])
def test_other_students_every_level_match_float64_port(kind):
    """MobileNetV2 and the full ESPNet, AT and MIMIC at all five levels (adapters sized from each network's level_channels(), e.g.
    MobileNetV2's 320-channel features[17] -> 2048) at 360x480, batch 2: one step's AT / MIMIC terms, task loss and adapter gradients
    against the same step of the students' plain-torch ports and the teacher in float64 on the GPU, the teacher's levels resampled
    onto the students' grids.  Bounds as tests/test_pa_levels_gpu.py's for these students, adapter gradients as test_step_matches_golden's."""
    from oracle import cases, espnet_full_port, feature_kd_port as P, mobilenet_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    lam_at, lam_mimic = [500.0] * 5, [1.0] * 5
    teacher, _, _ = cases.build_models(seed=0, with_D=False)
    ref = {"espnet": espnet_full_port, "mobilenetv2": mobilenet_port}[kind].build_student(7)
    m = NetModel(make_args(batch_size=2, pi=True, pa=False, ho=False, student=kind, at=True, lambda_at=lam_at, mimic=True,
                           lambda_mimic=lam_mimic))
    m.student.load_state_dict(ref.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    adapters = P.build_adapters(ref, teacher, lam_mimic, 4)
    m.mimic_adapters.load_state_dict(adapters.state_dict())
    if kind == "mobilenetv2":
        for d, mk in zip(m.student.dropouts(), cases.dropout_masks(ref, 2, seed=2)):
            d.injected = mk
        for d, mk in zip(ref.dropouts(), cases.dropout_masks(ref, 2, seed=2)):
            d.injected = mk.cuda()
    images, labels = port.synthetic_batch(2, 360, 480, seed=1)
    m.set_input((images, labels, None, None))
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    tf = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        refd, td, ad = ref.cuda().double(), teacher.cuda().double(), adapters.cuda().double()
        out = P.distill_step(kind, td, refd, None, ad, images.cuda().double(), labels.cuda(), port.StepConfig(pi=True, pa=False, ho=False),
                             at=lam_at, mimic=lam_mimic)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf
    rep = dict(ce=_relf(m.mc_G_loss, out["ce"]), pi=_relf(m.pi_G_loss, out["pi"]), G=_relf(m.G_loss, out["G"]))
    for term in ("at", "mimic"):
        for ind, (a, b) in enumerate(zip(getattr(m, term + "_G_loss"), out[term])):
            rep["%s%d" % (term, ind)] = _relf(a, b)
    mine = dict(m.mimic_adapters.named_parameters())
    for k, p in ad.named_parameters():
        rep["grad_" + k] = _rel(mine[k].grad.double(), p.grad)
    print("\nPARITY feature_kd", kind, {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        if k in ("ce", "pi", "G"):
            assert v < 1e-3, (k, v)
        elif k.startswith("mimic"):
            assert v < 5e-3, (k, v)
        elif k.startswith("at"):
            assert v < 1e-2, (k, v)
        else:
            assert v < 0.1, (k, v)


# -------------------------------------------------------------------------------------------- graphs, repeatability, state, ranks
GRAPH_CFG = dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")
GRAPH_EXTRA = dict(at=True, lambda_at=[500.0, 0.0, 500.0, 500.0, 500.0], mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0, 1.0],
                   overlap_streams=False)


def _terms(v):
    return [float(t) for t in v] if isinstance(v, list) else [float(v)]


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + _terms(m.at_G_loss) + _terms(m.mimic_G_loss) + \
        [p.detach().clone() for p in m.student.parameters()] + [p.detach().clone() for p in m.mimic_adapters.parameters()] + \
        [b.detach().clone() for b in m.student.buffers()]


def _same(a, b):
    return all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


def _state(m):
    return [{k: v.clone() for k, v in mod.state_dict().items()} for mod in (m.student, m.D_model, m.mimic_adapters)] + \
        [m.G_solver.flat_m.clone(), m.D_solver.flat_m.clone()]


def _rewind(m, snap):
    with torch.no_grad():
        for mod, sd in zip((m.student, m.D_model, m.mimic_adapters), snap[:3]):
            cur = mod.state_dict()
            for k, v in sd.items():
                cur[k].copy_(v)                                           # in place: the captured graph reads these buffers
        m.G_solver.flat_m.copy_(snap[3]); m.D_solver.flat_m.copy_(snap[4])


def test_cuda_graph_replays_equal_eager_and_runs_repeat():
    """ResNet18 Pi + Pa + Ho + four AT levels + MIMIC at x4 (512 -> 2048) and the PSP features, 360x480 batch 2, overlap_streams off:
    two eager runs of three steps are bitwise equal, and three replays of the captured step, rewound to the starting state, equal them."""
    runs = []
    for _ in range(2):
        m = _resnet18(2, 360, 480, GRAPH_CFG, **GRAPH_EXTRA)
        want = []
        for _ in range(3):
            m.optimize_parameters()
            torch.cuda.synchronize()
            want.append(_dump(m))
        runs.append(want)
        del m
    assert all(_same(a, b) for a, b in zip(*runs))
    m = _resnet18(2, 360, 480, GRAPH_CFG, **GRAPH_EXTRA)
    snap = _state(m)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()
    assert m._graphs["captured"]
    _rewind(m, snap)
    for w in runs[0]:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)


def test_training_state_keys_and_resume(tmp_path):
    """A MIMIC model's training state carries `mimic_state_dict`; one without MIMIC writes exactly the keys it always did.  Three steps,
    a save, a load into a fresh CUDA-graph model and three more steps equal six uninterrupted steps bit for bit."""
    extra = dict(at=True, lambda_at=500.0, mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0, 1.0])
    cfg = dict(pi=True, pa=True, ho=True, adv_type="hinge")
    plain = _resnet18(1, 256, 256, cfg)
    plain.save_training_state(str(tmp_path / "plain.pth"), 0)
    keys = set(torch.load(str(tmp_path / "plain.pth"), weights_only=False))
    assert keys == {"format", "version", "world_size", "kind", "classes_num", "step", "epoch", "best_mean_IU", "IU_array", "ranks",
                    "state_dict", "D_state_dict", "G_solver", "D_solver"}
    del plain
    want = []
    m = _resnet18(1, 256, 256, cfg, **extra)
    for k in range(6):
        m.optimize_parameters()
        if k == 2:
            m.save_training_state(str(tmp_path / "mimic.pth"), 3)
        if k >= 3:
            torch.cuda.synchronize()
            want.append(_dump(m))
    ck = torch.load(str(tmp_path / "mimic.pth"), weights_only=False)
    assert set(ck) == keys | {"mimic_state_dict"}
    assert set(ck["mimic_state_dict"]) == {"level3.weight", "level3.bias", "level4.weight", "level4.bias"}
    del m
    m = _resnet18(1, 256, 256, cfg, **extra)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                   # captured
    assert m._graphs["captured"]
    assert m.load_training_state(str(tmp_path / "mimic.pth")) == 3
    for w in want:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)
    other = _resnet18(1, 256, 256, cfg, at=True)
    with pytest.raises(ValueError, match="G_solver.numel|mimic_state_dict"):
        other.load_training_state(str(tmp_path / "mimic.pth"))


def test_defaults_launch_no_feature_kernel(monkeypatch):
    """With at / mimic off (make_args' defaults) no AT or MSE kernel runs, no adapter exists and G_solver holds the student alone."""
    from structure_knowledge_distillation_b200 import ops

    def refuse(*a, **k):
        raise AssertionError("a feature-distillation kernel ran with the terms off")
    for fn in ("at_fwd", "at_bwd", "mse_fwd", "mse_bwd"):
        monkeypatch.setattr(ops, fn, refuse)
    m = _resnet18(1, 256, 256, dict(pi=True, pa=True, ho=True, adv_type="wgan-gp"))
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert m.mimic_adapters is None and m.at_G_loss is None and m.mimic_G_loss is None
    trained = [p for p in m.student.parameters() if p.requires_grad]
    assert len(m.G_solver.params) == len(trained) and all(a is b for a, b in zip(m.G_solver.params, trained))


def _ddp_worker(rank, world, port, out):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port as oport
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        torch.manual_seed(100 + rank)                                  # different init per rank: NetModel broadcasts rank 0's
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, at=True,
                               lambda_at=[500.0] * 5, mimic=True, lambda_mimic=[0.0, 0.0, 1.0, 1.0, 1.0]))
        for d in m.student.dropouts():
            d.injected = (torch.rand(1, 128, generator=torch.Generator().manual_seed(5 + rank)) >= 0.1).float()
        images, labels = oport.synthetic_batch(1, 360, 480, seed=7 + rank)          # each rank its own shard
        m.set_input((images, labels, None, None))
        m.G_solver._buckets = None                                                   # one exchange after backward
        m._student_phase()
        local = m.G_solver.flat_g.clone()
        m.G_solver.all_reduce_grads(world)
        summed = m.G_solver.flat_g.clone()
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        ref_sum = sum(parts)
        err = float((summed - ref_sum).norm() / ref_sum.norm())
        assert err < 1e-6, err
        lo = m.G_solver._offsets[sum(1 for p in m.student.parameters() if p.requires_grad)]   # the adapters follow the student
        ad_err = float((summed[lo:] - ref_sum[lo:]).norm() / ref_sum[lo:].norm())
        if rank == 0:
            out.put(("ok", err, ad_err, [float(v) for v in m.mimic_G_loss]))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_sums_the_shard_gradients():
    """ResNet18 with AT at five levels and MIMIC at three over 2 NCCL ranks: the all-reduced flat gradient (adapters included) is the
    sum of the per-rank gradients.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29643, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY feature_kd world2", res)
    assert res[0] == "ok" and res[2] < 1e-6, res
