"""Intra-class feature variation distillation on the host: the restatement (oracle/ifv_port.py, IFVD's per-class loop) against an
independent index_add form in float64, torch's zero-vector cosine, the nearest rule the label kernel implements against F.interpolate,
the fixture against its generator, NetModel's validation of the options before any device work, the defaults and the log line."""
import logging
import math
import types

import pytest
import torch
import torch.nn.functional as F


def _maps(n, cs, ct, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, cs, h, w, generator=g, dtype=torch.float64), torch.randn(n, ct, h, w, generator=g, dtype=torch.float64), g)


def _both(S, T, labels, K):
    """(loss, dS) of the loop form and of the index_add form."""
    from oracle import ifv_port as P
    out = []
    for fn in (P.ifv_loss, P.ifv_loss_scatter):
        s = S.clone().requires_grad_(True)
        loss = fn(s, T, labels, K)
        (g,) = torch.autograd.grad(loss, s)
        out.append((float(loss), g))
    return out


@pytest.mark.parametrize("n, cs, ct, h, w, H, W, K", [(2, 5, 7, 9, 11, 33, 41, 4), (1, 3, 6, 5, 5, 17, 17, 19), (3, 8, 8, 7, 9, 20, 24, 150),
                                                      (2, 16, 4, 13, 17, 104, 136, 21)])
def test_loop_matches_index_add_restatement(n, cs, ct, h, w, H, W, K):
    S, T, g = _maps(n, cs, ct, h, w, n + cs + K)
    labels = torch.randint(0, K, (n, H, W), generator=g)
    labels[torch.rand(n, H, W, generator=g) < 0.1] = 255
    (l1, g1), (l2, g2) = _both(S, T, labels, K)
    assert l1 == pytest.approx(l2, rel=1e-12) and torch.allclose(g1, g2, rtol=1e-10, atol=1e-16)


def test_edge_cases_absent_class_all_ignored_image_one_pixel_class_zero_vector():
    """Classes 5.. absent, image 1 all ignored, class 4 on exactly one pixel, an all-zero student pixel: both forms agree, the ignored
    image gets exactly zero gradient, and a one-pixel class has cos = 1 in both maps (d = 0, no loss from it)."""
    n, cs, ct, h, w, K = 2, 6, 10, 6, 8, 19
    S, T, g = _maps(n, cs, ct, h, w, 3)
    labels = torch.randint(0, 4, (n, h, w), generator=g)
    labels[1] = 255
    labels[0, 2, 3] = 4
    S[0, :, 4, 4] = 0.0
    (l1, g1), (l2, g2) = _both(S, T, labels, K)
    assert l1 == pytest.approx(l2, rel=1e-12) and torch.allclose(g1, g2, rtol=1e-10, atol=1e-16)
    assert torch.count_nonzero(g1[1]) == 0
    assert float(g1[0, :, 4, 4].norm()) > 1e5                      # p_hat / eps at the zero vector (torch's cosine_similarity)
    from oracle import ifv_port as P
    one = torch.full((1, 1, 1), 4)
    assert float(P.ifv_loss(S[:1, :, 2:3, 3:4], T[:1, :, 2:3, 3:4], one, K)) == pytest.approx(0.0, abs=1e-24)


def test_zero_vector_follows_torch_cosine_similarity():
    """torch gives cos = 0 for an all-zero f and the gradient p / |p| / eps: the value the kernels follow."""
    p = torch.tensor([[3.0, 4.0]], dtype=torch.float64)
    f = torch.zeros(1, 2, dtype=torch.float64, requires_grad=True)
    c = F.cosine_similarity(f, p, dim=1)
    (g,) = torch.autograd.grad(c.sum(), f)
    assert float(c) == 0.0 and torch.allclose(g, p / 5.0 / 1e-8, rtol=1e-12)


def _nearest(labels, h, w):
    """The rule ops.labels_nearest implements: src = min(floor(dst * (float(in) / out)), in - 1), product and quotient in fp32."""
    H, W = labels.shape[-2:]
    sy, sx = torch.tensor(H, dtype=torch.float32) / h, torch.tensor(W, dtype=torch.float32) / w
    ys = torch.clamp(torch.floor(torch.arange(h, dtype=torch.float32) * sy).long(), max=H - 1)
    xs = torch.clamp(torch.floor(torch.arange(w, dtype=torch.float32) * sx).long(), max=W - 1)
    return labels[:, ys][:, :, xs]


@pytest.mark.parametrize("H, W, h, w", [(512, 512, 65, 65), (512, 1024, 65, 129), (512, 1024, 129, 257), (769, 769, 97, 97),
                                        (360, 480, 45, 60), (360, 480, 46, 61)])
def test_nearest_rule_matches_interpolate_at_the_students_grids(H, W, h, w):
    g = torch.Generator().manual_seed(H + w)
    labels = torch.randint(0, 256, (2, H, W), generator=g)
    want = F.interpolate(labels[:, None].float(), (h, w), mode="nearest")[:, 0].long()
    assert torch.equal(_nearest(labels, h, w), want)


def test_nearest_rule_random_sweep():
    g = torch.Generator().manual_seed(9)
    for _ in range(200):
        H, W = (int(v) for v in torch.randint(1, 2100, (2,), generator=g))
        h, w = (int(v) for v in torch.randint(1, 400, (2,), generator=g))
        labels = torch.randint(0, 256, (1, H, W), generator=g)
        want = F.interpolate(labels[:, None].float(), (h, w), mode="nearest")[:, 0].long()
        assert torch.equal(_nearest(labels, h, w), want), (H, W, h, w)


@pytest.fixture(scope="module")
def golden():
    from oracle import make_golden_ifv as G
    return G.load()


CASES = ["r18_pi_pa_ho_ifv_psp_512_b1", "r18_ifv_levels_cwd_96x128_b2", "espnet_c_ifv_psp_360x480_b1", "mbv2_ifv_psp_voc21_96x128_b2"]


@pytest.mark.parametrize("name", CASES)
def test_fixture_reproduces_from_its_generator(golden, name):
    """The generator's step on the CPU reproduces the stored record (thread counts may reorder fp32 sums: 1e-4)."""
    from oracle import feature_kd_port as FK, make_golden_ifv as G
    gold, mine = golden[name], G.port_step(G.GOLDEN_CASES[name])
    for k in ("ce", "pi", "pa", "adv_g", "G", "D", "cwd", "ifv"):
        if k in gold:
            a, b = (mine[k], gold[k]) if isinstance(gold[k], list) else ([mine[k]], [gold[k]])
            assert a == pytest.approx(b, rel=1e-4, abs=1e-12), k
    assert torch.allclose(mine["logits_S"], gold["logits_S"], rtol=1e-3, atol=1e-4)
    for k, v in gold["student_grads"].items():
        assert mine["student_grads"][k]["norm"] == pytest.approx(v["norm"], rel=1e-3, abs=1e-9), k
    spec = G.GOLDEN_CASES[name]
    ifv = gold["ifv"] if isinstance(gold["ifv"], list) else [gold["ifv"]]
    assert len(ifv) == len(FK.levels(spec["ifv"])) and all(v > 0 for v in ifv)


@pytest.mark.parametrize("kw, match", [
    (dict(ifv="yes"), "ifv must be True or False"),
    (dict(ifv=2), "ifv must be True or False"),
    (dict(lambda_ifv=-1.0, ifv=True), "lambda_ifv must be finite and >= 0"),
    (dict(lambda_ifv=math.nan), "lambda_ifv must be finite"),
    (dict(lambda_ifv=math.inf, ifv=True), "lambda_ifv must be finite"),
    (dict(lambda_ifv="x"), "lambda_ifv must be a number"),
    (dict(lambda_ifv=[], ifv=True), "lambda_ifv list must have 1..5 entries"),
    (dict(lambda_ifv=[1.0] * 6), "lambda_ifv list must have 1..5 entries"),
    (dict(lambda_ifv=[1.0, -0.5], ifv=True), "IFV level 1: lambda_ifv must be finite and >= 0"),
    (dict(lambda_ifv=[math.nan]), "IFV level 0: lambda_ifv must be finite"),
    (dict(lambda_ifv=["x"], ifv=True), "IFV level 0: lambda_ifv must be a number"),
])
def test_netmodel_rejects_bad_options_before_device_work(kw, match):
    """ValueError from NetModel's constructor, with ifv on or off, before it looks for a device (this runs without one)."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    with pytest.raises(ValueError, match=match):
        NetModel(make_args(**kw))


def test_ops_refuse_mismatched_inputs():
    """Student / teacher maps on different batches or grids, labels that are not contiguous (N, H, W) int64 or hold another batch, and
    class counts outside [1, 255] are refused before any launch.  Different widths are allowed."""
    from structure_knowledge_distillation_b200 import ops
    S, lab = torch.zeros(2, 3, 4, 5), torch.zeros(2, 32, 40, dtype=torch.long)
    ops._ifv_check(S, torch.zeros(2, 7, 4, 5), lab, 19)
    for T in (torch.zeros(1, 3, 4, 5), torch.zeros(2, 3, 4, 6), torch.zeros(2, 3, 5, 5)):
        with pytest.raises(ValueError, match="differ in batch or grid"):
            ops._ifv_check(S, T, lab, 19)
    for bad in (lab.int(), lab.float(), lab[:, :, ::2], lab[:, None]):
        with pytest.raises(ValueError, match="labels must be a contiguous"):
            ops._ifv_check(S, S, bad, 19)
    with pytest.raises(ValueError, match="labels hold 1 images for a batch of 2"):
        ops._ifv_check(S, S, lab[:1], 19)
    for k in (0, 256, -1):
        with pytest.raises(ValueError, match="class count"):
            ops._ifv_check(S, S, lab, k)


def test_criterion_refuses_an_ignore_index_inside_the_classes():
    from structure_knowledge_distillation_b200.utils.criterion import CriterionIFV
    assert CriterionIFV(-5, 19).ignore_index == 255
    with pytest.raises(ValueError, match="ignore_index 3"):
        CriterionIFV(-5, 19, ignore_index=3)
    with pytest.raises(ValueError, match="classes_num"):
        CriterionIFV(-5, 300)


def test_make_args_leaves_ifv_off():
    from structure_knowledge_distillation_b200.utils.criterion import check_ifv_args
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args()
    assert a.ifv is False and a.lambda_ifv == 200.0
    assert check_ifv_args(a) == []
    assert check_ifv_args(make_args(ifv=True)) == [(-5, 200.0)]
    assert check_ifv_args(make_args(ifv=True, lambda_ifv=[0, 1.5])) == [(-1, 0.0), (-2, 1.5)]


def test_print_info_appends_ifv_only_when_on(caplog):
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.step_model import _LazyScalar
    groups = types.SimpleNamespace(param_groups=[{"lr": 0.01}])
    m = types.SimpleNamespace(G_solver=groups, D_solver=groups, G_loss=_LazyScalar(torch.tensor(3.0)), mc_G_loss=1.0, pi_G_loss=2.0,
                              pa_G_loss=0.25, D_loss=0.5, at_G_loss=None, mimic_G_loss=None, cwd_G_loss=None, ifv_G_loss=None)
    with caplog.at_level(logging.INFO):
        NetModel.print_info(m, 0, 7)
        m.ifv_G_loss = _LazyScalar(torch.tensor(0.375))
        NetModel.print_info(m, 0, 8)
        m.cwd_G_loss, m.ifv_G_loss = 0.5, [_LazyScalar(torch.tensor(0.25)), 0.0, 0.125]
        NetModel.print_info(m, 0, 9)
    assert caplog.records[0].getMessage() == ("step:    7 G_lr:0.010000 G_loss:3.00000(mc:1.00000 pixelwise:2.00000 pairwise:0.25000) "
                                              "D_lr:0.010000 D_loss:0.50000")
    assert "pairwise:0.25000 ifv:0.37500) D_lr" in caplog.records[1].getMessage()
    assert "pairwise:0.25000 cwd:0.50000 ifv:[0.25000, 0.00000, 0.12500]) D_lr" in caplog.records[2].getMessage()
