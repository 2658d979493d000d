"""Attention transfer and MIMIC on the host: the restatement (oracle/feature_kd_port.py) against the formulas evaluated directly in
float64, the fixture against its generator, NetModel's validation of the options before any device work, the level order and the log
line."""
import logging
import math
import types

import pytest
import torch


def _direct_at(S, T):
    """L = mean over N*H*W of (q^_S - q^_T)^2, q = mean_c a_c^2, q^ = q / max(||q||_2, 1e-12), written out pixel by pixel."""
    n = S.shape[0]
    total = 0.0
    for i in range(n):
        qs = [[float((S[i, :, y, x] ** 2).sum()) / S.shape[1] for x in range(S.shape[3])] for y in range(S.shape[2])]
        qt = [[float((T[i, :, y, x] ** 2).sum()) / T.shape[1] for x in range(T.shape[3])] for y in range(T.shape[2])]
        ns = max(math.sqrt(sum(v * v for r in qs for v in r)), 1e-12)
        nt = max(math.sqrt(sum(v * v for r in qt for v in r)), 1e-12)
        total += sum((a / ns - b / nt) ** 2 for ra, rb in zip(qs, qt) for a, b in zip(ra, rb))
    return total / (n * S.shape[2] * S.shape[3])


@pytest.mark.parametrize("zero", [False, True])
def test_at_restatement_matches_the_formula(zero):
    from oracle import feature_kd_port as P
    g = torch.Generator().manual_seed(1)
    S = torch.randn(3, 5, 7, 9, generator=g, dtype=torch.float64)
    T = torch.randn(3, 11, 7, 9, generator=g, dtype=torch.float64)
    if zero:
        S[1].zero_()                                           # the clamp branch: q = 0, ||q|| clamped to 1e-12
    assert float(P.at_loss(S, T)) == pytest.approx(_direct_at(S, T), rel=1e-12)
    Sg = S.clone().requires_grad_(True)
    P.at_loss(Sg, T).backward()
    if zero:
        assert torch.count_nonzero(Sg.grad[1]) == 0
    # gradient: dL/da = (2/C) a g with g = (h - q^ <q^, h>) / ||q||, h = 2 (q^_S - q^_T) / (N H W)
    q = S.pow(2).mean(1).flatten(1)
    nrm = q.norm(dim=1, keepdim=True)
    qs, qt = q / nrm.clamp_min(1e-12), P.at_map(T)
    h = 2 * (qs - qt) / q.numel()
    gq = torch.where(nrm >= 1e-12, (h - qs * (qs * h).sum(1, keepdim=True)) / nrm.clamp_min(1e-12), h / 1e-12)
    want = 2.0 / S.shape[1] * S * gq.view(3, 1, 7, 9)
    assert torch.allclose(Sg.grad, want, rtol=1e-10, atol=1e-300)


def test_mimic_restatement_matches_the_formula():
    from oracle import feature_kd_port as P
    g = torch.Generator().manual_seed(2)
    S = torch.randn(2, 6, 5, 7, generator=g, dtype=torch.float64)
    T = torch.randn(2, 10, 5, 7, generator=g, dtype=torch.float64)
    conv = torch.nn.Conv2d(6, 10, 1).double()
    r = torch.einsum("oc,nchw->nohw", conv.weight[:, :, 0, 0], S) + conv.bias.view(1, -1, 1, 1)
    assert float(P.mimic_loss(S, T, conv)) == pytest.approx(float(((r - T) ** 2).sum()) / T.numel(), rel=1e-12)


def test_levels_follow_the_pair_wise_order():
    from oracle import feature_kd_port as P
    from structure_knowledge_distillation_b200.networks.kd_model import mimic_adapters
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    from structure_knowledge_distillation_b200.utils.criterion import (CriterionAT, check_feature_levels, feature_level_criteria)
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    assert check_feature_levels(make_args(), "lambda_at", "attention-transfer", 500.0) == [(-5, 500.0)]
    lv = check_feature_levels(make_args(lambda_at=(1, 0.0, 2.5)), "lambda_at", "attention-transfer", 500.0)
    assert lv == [(-1, 1.0), (-2, 0.0), (-3, 2.5)]
    crits = feature_level_criteria(lv, CriterionAT)
    assert crits[1] is None and [c.feat_ind for c in (crits[0], crits[2])] == [-1, -3]
    assert P.levels([1.0, 0.0, 2.5]) == lv
    ad = mimic_adapters(build_seg_network("resnet18", 19), build_seg_network("resnet101", 19),
                        [(-1, 0.0), (-2, 0.0), (-3, 0.0), (-4, 1.0), (-5, 1.0)])
    assert {k: tuple(v.shape) for k, v in ad.state_dict().items()} == {
        "level3.weight": (2048, 512, 1, 1), "level3.bias": (2048,), "level4.weight": (512, 128, 1, 1), "level4.bias": (512,)}
    assert ad["level3"].weight.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("kind", ["resnet101", "resnet18", "espnet_c", "espnet", "mobilenetv2"])
def test_level_channels_are_the_networks_widths(kind):
    """level_channels() of every network NetModel trains or distils from, which sizes the MIMIC adapters, equals the channel counts of
    preds[-1] .. preds[-5] that its plain-torch port's forward produces; so every student's adapter at every level fits its input."""
    from oracle import espnet_full_port, espnet_port, feature_kd_port as P, mobilenet_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import mimic_adapters
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    ports = {"resnet101": lambda: port.PSPNet("resnet101", 19), "resnet18": lambda: port.PSPNet("resnet18", 19),
             "espnet_c": lambda: espnet_port.build_student(7), "espnet": lambda: espnet_full_port.build_student(7),
             "mobilenetv2": lambda: mobilenet_port.build_student(7)}
    net, ref = build_seg_network(kind, 19), ports[kind]()
    widths = P.level_channels(ref)
    assert net.level_channels() == widths, (kind, net.level_channels(), widths)
    teacher = build_seg_network("resnet101", 19)
    ad = mimic_adapters(net, teacher, [(-(ind + 1), 1.0) for ind in range(5)])
    tw = teacher.level_channels()
    assert {k: tuple(m.weight.shape) for k, m in ad.items()} == {"level%d" % ind: (tw[ind], widths[ind], 1, 1)
                                                                   for ind in range(5)}


@pytest.fixture(scope="module")
def golden():
    from oracle import make_golden_feature_kd as G
    return G.load()


@pytest.mark.parametrize("name", ["r18_pi_pa_ho_at_mimic_psp_512_b1", "r18_at5_mimic_x3_96x128_b2", "espnet_c_at5_mimic_psp_360x480_b1"])
def test_fixture_reproduces_from_its_generator(golden, name):
    """The generator's step on the CPU reproduces the stored record (thread counts may reorder fp32 sums: 1e-4)."""
    from oracle import feature_kd_port as P, make_golden_feature_kd as G
    gold, mine = golden[name], G.port_step(G.GOLDEN_CASES[name])
    for k in ("ce", "pi", "pa", "adv_g", "G", "D", "at", "mimic"):
        if k in gold:
            a, b = (mine[k], gold[k]) if isinstance(gold[k], list) else ([mine[k]], [gold[k]])
            assert a == pytest.approx(b, rel=1e-4, abs=1e-12), k
    assert torch.allclose(mine["logits_S"], gold["logits_S"], rtol=1e-3, atol=1e-4)
    for part in ("student_grads", "adapter_grads"):
        for k, v in gold[part].items():
            assert mine[part][k]["norm"] == pytest.approx(v["norm"], rel=1e-3, abs=1e-9), (part, k)
    spec = G.GOLDEN_CASES[name]
    for term in ("at", "mimic"):
        w = spec[term]
        if isinstance(w, list):                                     # a zero weight logs 0.0, the others a term
            assert len(gold[term]) == len(w) and all((v == 0.0) == (l == 0.0) for v, l in zip(gold[term], w))
    assert set(gold["adapter_grads"]) == {"level%d.%s" % (-i - 1, p) for i, w in P.levels(spec["mimic"]) if w for p in ("weight", "bias")}


@pytest.mark.parametrize("kw, match", [
    (dict(lambda_at=-1.0), "lambda_at must be finite and >= 0"),
    (dict(lambda_at=math.nan, at=True), "lambda_at must be finite"),
    (dict(lambda_mimic=math.inf, mimic=True), "lambda_mimic must be finite"),
    (dict(lambda_at=[], at=True), "lambda_at list must have 1..5 entries"),
    (dict(lambda_mimic=[1.0] * 6, mimic=True), "lambda_mimic list must have 1..5 entries"),
    (dict(lambda_at=[1.0, -0.5], at=True), "attention-transfer level 1: lambda_at must be finite and >= 0"),
    (dict(lambda_mimic=[math.nan], mimic=True), "MIMIC level 0: lambda_mimic must be finite"),
    (dict(lambda_mimic=["x"], mimic=True), "MIMIC level 0: lambda_mimic must be a number"),
    (dict(lambda_at="x"), "lambda_at must be a number"),
])
def test_netmodel_rejects_bad_weights_before_device_work(kw, match):
    """ValueError from NetModel's constructor, before it looks for a device (this runs without one)."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    with pytest.raises(ValueError, match=match):
        NetModel(make_args(**kw))


def test_make_args_leaves_the_terms_off():
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args()
    assert a.at is False and a.mimic is False and a.lambda_at == 500.0 and a.lambda_mimic == 1.0


def test_print_info_appends_the_terms_only_when_on(caplog):
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.step_model import _LazyScalar
    groups = types.SimpleNamespace(param_groups=[{"lr": 0.01}])
    m = types.SimpleNamespace(G_solver=groups, D_solver=groups, G_loss=_LazyScalar(torch.tensor(3.0)), mc_G_loss=1.0, pi_G_loss=2.0,
                              pa_G_loss=0.25, D_loss=0.5, at_G_loss=None, mimic_G_loss=None)
    with caplog.at_level(logging.INFO):
        NetModel.print_info(m, 0, 7)
        m.at_G_loss, m.mimic_G_loss = _LazyScalar(torch.tensor(0.125)), [0.0, _LazyScalar(torch.tensor(0.5))]
        NetModel.print_info(m, 0, 8)
    assert caplog.records[0].getMessage() == ("step:    7 G_lr:0.010000 G_loss:3.00000(mc:1.00000 pixelwise:2.00000 pairwise:0.25000) "
                                              "D_lr:0.010000 D_loss:0.50000")
    assert "pairwise:0.25000 at:0.12500 mimic:[0.00000, 0.50000]) D_lr" in caplog.records[1].getMessage()
