"""Channel-wise distillation on the host: the restatement (oracle/cwd_port.py) against the F.kl_div formula in float64, including a map
whose softmax underflows, the fixture against its generator, NetModel's validation of the options before any device work, the defaults
and the log line."""
import logging
import math
import types

import pytest
import torch
import torch.nn.functional as F


def _kl_div(S, T, tau):
    """tau^2 * F.kl_div(log_softmax(S / tau), log_softmax(T / tau), log_target=True, reduction='sum') / (N*C) over flattened H*W."""
    n, c = S.shape[:2]
    return tau ** 2 * F.kl_div(F.log_softmax(S.flatten(2) / tau, -1), F.log_softmax(T.flatten(2) / tau, -1), log_target=True,
                               reduction="sum") / (n * c)


@pytest.mark.parametrize("shape, tau", [((2, 3, 5, 7), 4.0), ((1, 19, 9, 11), 1.0), ((3, 1, 1, 1), 4.0), ((2, 4, 1, 13), 0.5)])
def test_restatement_matches_kl_div(shape, tau):
    from oracle import cwd_port as P
    g = torch.Generator().manual_seed(sum(shape))
    S = torch.randn(*shape, generator=g, dtype=torch.float64) * 3
    T = torch.randn(*shape, generator=g, dtype=torch.float64) * 3
    Sg = S.clone().requires_grad_(True)
    loss = P.cwd_loss(Sg, T, tau)
    assert float(loss) == pytest.approx(float(_kl_div(S, T, tau)), rel=1e-12, abs=1e-15)
    loss.backward()
    # dL/dS = tau / (N*C) * (pS - pT)
    n, c = shape[:2]
    ps, pt = F.softmax(S.flatten(2) / tau, -1), F.softmax(T.flatten(2) / tau, -1)
    assert torch.allclose(Sg.grad, (tau / (n * c) * (ps - pt)).view(shape), rtol=1e-10, atol=1e-15)


def test_restatement_stays_finite_where_softmax_log_underflows():
    """Logits x1000 at tau = 1: softmax(S).log() is -inf (exp underflows in float64) at positions far below the channel's maximum, so
    the naive loss is inf; the log_softmax form stays finite and equals F.kl_div's."""
    from oracle import cwd_port as P
    g = torch.Generator().manual_seed(3)
    S = torch.randn(2, 3, 6, 8, generator=g, dtype=torch.float64) * 1000
    T = torch.randn(2, 3, 6, 8, generator=g, dtype=torch.float64) * 1000
    ps_log = F.softmax(S.flatten(2), -1).log()
    pt = F.softmax(T.flatten(2), -1)
    naive = (pt * (pt.log() - ps_log)).sum() / 6
    assert torch.isinf(ps_log).any() and not math.isfinite(float(naive))
    loss = P.cwd_loss(S, T, 1.0)
    assert math.isfinite(float(loss)) and float(loss) == pytest.approx(float(_kl_div(S, T, 1.0)), rel=1e-12)


def test_equal_maps_and_single_pixel_give_zero():
    from oracle import cwd_port as P
    g = torch.Generator().manual_seed(4)
    S = torch.randn(2, 5, 4, 3, generator=g, dtype=torch.float64)
    assert float(P.cwd_loss(S, S.clone(), 4.0)) == 0.0
    assert float(P.cwd_loss(torch.randn(3, 7, 1, 1, dtype=torch.float64), torch.randn(3, 7, 1, 1, dtype=torch.float64), 4.0)) == 0.0


@pytest.fixture(scope="module")
def golden():
    from oracle import make_golden_cwd as G
    return G.load()


CASES = ["r18_pi_pa_ho_cwd_logits_512_b1", "r18_cwd_levels_mimic_x3_96x128_b2", "espnet_cwd_logits_360x480_b1",
         "espnet_c_cwd_psp_360x480_b1"]


@pytest.mark.parametrize("name", CASES)
def test_fixture_reproduces_from_its_generator(golden, name):
    """The generator's step on the CPU reproduces the stored record (thread counts may reorder fp32 sums: 1e-4)."""
    from oracle import feature_kd_port as FK, make_golden_cwd as G
    gold, mine = golden[name], G.port_step(G.GOLDEN_CASES[name])
    for k in ("ce", "pi", "pa", "adv_g", "G", "D", "mimic", "cwd"):
        if k in gold:
            a, b = (mine[k], gold[k]) if isinstance(gold[k], list) else ([mine[k]], [gold[k]])
            assert a == pytest.approx(b, rel=1e-4, abs=1e-12), k
    assert torch.allclose(mine["logits_S"], gold["logits_S"], rtol=1e-3, atol=1e-4)
    for part in ("student_grads", "mimic_adapter_grads", "cwd_adapter_grads"):
        for k, v in gold[part].items():
            assert mine[part][k]["norm"] == pytest.approx(v["norm"], rel=1e-3, abs=1e-9), (part, k)
    spec = G.GOLDEN_CASES[name]
    if spec["cwd_feat"] is None:
        assert not isinstance(gold["cwd"], list) and gold["cwd"] > 0
    else:
        assert len(gold["cwd"]) == 1 + len(FK.levels(spec["cwd_feat"]))
        assert (gold["cwd"][0] == 0.0) == (spec["lambda_cwd"] == 0.0)
    for fam, w in (("mimic", spec["mimic"]), ("cwd", spec["cwd_feat"])):
        assert set(gold[fam + "_adapter_grads"]) == {"level%d.%s" % (-i - 1, p) for i, l in FK.levels(w) if l for p in ("weight", "bias")}


@pytest.mark.parametrize("kw, match", [
    (dict(cwd_tau=0.0), "cwd_tau must be finite and > 0"),
    (dict(cwd_tau=-1.0, cwd=True), "cwd_tau must be finite and > 0"),
    (dict(cwd_tau=math.inf, cwd=True), "cwd_tau must be finite"),
    (dict(cwd_tau=math.nan), "cwd_tau must be finite"),
    (dict(cwd_tau="x"), "cwd_tau must be a number"),
    (dict(lambda_cwd=[1.0, 2.0], cwd=True), "lambda_cwd must be a number"),
    (dict(lambda_cwd=-1.0), "lambda_cwd must be finite and >= 0"),
    (dict(lambda_cwd=math.nan, cwd=True), "lambda_cwd must be finite"),
    (dict(lambda_cwd=math.inf), "lambda_cwd must be finite"),
    (dict(lambda_cwd_feat=-1.0, cwd=True), "lambda_cwd_feat must be finite and >= 0"),
    (dict(lambda_cwd_feat="x"), "lambda_cwd_feat must be a number"),
    (dict(lambda_cwd_feat=[], cwd=True), "lambda_cwd_feat list must have 1..5 entries"),
    (dict(lambda_cwd_feat=[1.0] * 6), "lambda_cwd_feat list must have 1..5 entries"),
    (dict(lambda_cwd_feat=[1.0, -0.5], cwd=True), "CWD level 1: lambda_cwd_feat must be finite and >= 0"),
    (dict(lambda_cwd_feat=[math.nan]), "CWD level 0: lambda_cwd_feat must be finite"),
    (dict(lambda_cwd_feat=["x"], cwd=True), "CWD level 0: lambda_cwd_feat must be a number"),
])
def test_netmodel_rejects_bad_options_before_device_work(kw, match):
    """ValueError from NetModel's constructor, with cwd on or off, before it looks for a device (this runs without one)."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    with pytest.raises(ValueError, match=match):
        NetModel(make_args(**kw))


def test_ops_refuse_mismatched_maps():
    """A student / teacher pair on different batches, grids or widths, or a bad temperature, is refused before any launch."""
    from structure_knowledge_distillation_b200 import ops
    S = torch.zeros(2, 3, 4, 5)
    for T in (torch.zeros(1, 3, 4, 5), torch.zeros(2, 3, 4, 6), torch.zeros(2, 4, 4, 5)):
        with pytest.raises(ValueError, match="differ in batch, channels or grid"):
            ops._cwd_check(S, T, 4.0)
    for tau in (0.0, -2.0, math.nan, math.inf):
        with pytest.raises(ValueError, match="temperature"):
            ops._cwd_check(S, S, tau)


def test_make_args_leaves_cwd_off():
    from structure_knowledge_distillation_b200.utils.criterion import check_cwd_args
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args()
    assert a.cwd is False and a.lambda_cwd == 3.0 and a.lambda_cwd_feat is None and a.cwd_tau == 4.0
    assert check_cwd_args(a) == (3.0, 4.0, [])
    assert check_cwd_args(make_args(lambda_cwd_feat=2.0)) == (3.0, 4.0, [(-5, 2.0)])
    assert check_cwd_args(make_args(lambda_cwd_feat=[0, 1.5], cwd_tau=2)) == (3.0, 2.0, [(-1, 0.0), (-2, 1.5)])


def test_print_info_appends_cwd_only_when_on(caplog):
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.step_model import _LazyScalar
    groups = types.SimpleNamespace(param_groups=[{"lr": 0.01}])
    m = types.SimpleNamespace(G_solver=groups, D_solver=groups, G_loss=_LazyScalar(torch.tensor(3.0)), mc_G_loss=1.0, pi_G_loss=2.0,
                              pa_G_loss=0.25, D_loss=0.5, at_G_loss=None, mimic_G_loss=None, cwd_G_loss=None)
    with caplog.at_level(logging.INFO):
        NetModel.print_info(m, 0, 7)
        m.cwd_G_loss = _LazyScalar(torch.tensor(0.375))
        NetModel.print_info(m, 0, 8)
        m.mimic_G_loss, m.cwd_G_loss = 0.5, [_LazyScalar(torch.tensor(0.25)), 0.0, 0.125]
        NetModel.print_info(m, 0, 9)
    assert caplog.records[0].getMessage() == ("step:    7 G_lr:0.010000 G_loss:3.00000(mc:1.00000 pixelwise:2.00000 pairwise:0.25000) "
                                              "D_lr:0.010000 D_loss:0.50000")
    assert "pairwise:0.25000 cwd:0.37500) D_lr" in caplog.records[1].getMessage()
    assert "pairwise:0.25000 mimic:0.50000 cwd:[0.25000, 0.00000, 0.12500]) D_lr" in caplog.records[2].getMessage()
