"""Local pair-wise distillation on the host: the restatement (oracle/pa_local_port.py) against the fully connected term when the window
covers the grid, its pair count against brute force, gradcheck, the fixture against its generator, NetModel's validation of pa_window /
pa_dilation before any device work, and the defaults building the criteria they always built."""
import itertools

import pytest
import torch


def _global_pooled(ps, pt):
    """The fully connected term of oracle/port.py on already pooled maps (port.pairwise_loss after its max pool)."""
    from oracle import port
    nodes = ps.shape[2] * ps.shape[3]
    return ((port.affinity(pt) - port.affinity(ps)) ** 2).sum() / nodes ** 2 / ps.shape[0]


def _covering(h, w):
    k = max(3, 2 * max(h, w) - 1)
    return k + (k % 2 == 0)


@pytest.mark.parametrize("h, w", [(1, 9), (9, 1), (1, 2), (2, 1), (5, 6), (9, 4), (3, 3), (7, 12)])
def test_covering_window_is_the_global_term(h, w):
    """d = 1 and r >= max(h, w) - 1: P = nodes^2 and the loss and its gradient are the fully connected term's, in float64 to 1e-12."""
    from oracle import pa_local_port as P
    g = torch.Generator().manual_seed(h * 31 + w)
    S = torch.randn(2, 5, h, w, generator=g, dtype=torch.float64, requires_grad=True)
    T = torch.randn(2, 3, h, w, generator=g, dtype=torch.float64)
    k = _covering(h, w)
    assert P.pair_count(h, w, k, 1) == (h * w) ** 2
    a, b = P.local_affinity_loss(S, T, k, 1), _global_pooled(S, T)
    (ga,), (gb,) = torch.autograd.grad(a, S), torch.autograd.grad(b, S)
    assert abs(float(a) - float(b)) <= 1e-12 * abs(float(b))
    assert float((ga - gb).norm()) <= 1e-12 * float(gb.norm())


@pytest.mark.parametrize("H, W, scale", [(12, 24, 0.25), (20, 13, 0.15), (8, 8, 0.5), (30, 50, 0.1)])
def test_covering_window_equals_port_pairwise_loss(H, W, scale):
    """Through the max pool too: pairwise_local_loss with a covering window equals oracle.port.pairwise_loss, loss and feature gradient."""
    from oracle import pa_local_port as P, port
    g = torch.Generator().manual_seed(H + W)
    S = torch.randn(2, 6, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    T = torch.randn(2, 4, H, W, generator=g, dtype=torch.float64)
    ph, pw = port.pool_patch(H, W, scale)
    h, w = -(-H // ph), -(-W // pw)
    a, b = P.pairwise_local_loss(S, T, scale, _covering(h, w), 1), port.pairwise_loss(S, T, scale)
    (ga,), (gb,) = torch.autograd.grad(a, S), torch.autograd.grad(b, S)
    assert abs(float(a) - float(b)) <= 1e-12 * abs(float(b))
    assert float((ga - gb).norm()) <= 1e-12 * float(gb.norm())


def _brute_pairs(h, w, k, d):
    r = (k - 1) // 2
    return sum(1 for y, x, t, u in itertools.product(range(h), range(w), range(-r, r + 1), range(-r, r + 1))
               if 0 <= y + t * d < h and 0 <= x + u * d < w)


@pytest.mark.parametrize("h, w, k, d", [(1, 1, 3, 1), (1, 17, 5, 2), (13, 1, 15, 1), (9, 7, 3, 1), (9, 7, 9, 2), (20, 11, 7, 4),
                                        (6, 30, 15, 8), (33, 5, 11, 3), (4, 4, 15, 1)])
def test_pair_count_matches_brute_force(h, w, k, d):
    from oracle import pa_local_port as P
    assert P.pair_count(h, w, k, d) == _brute_pairs(h, w, k, d)


def test_loss_matches_the_pair_by_pair_definition():
    """A small grid written out pair by pair: sum over i and j in W(i) of (a^T_ij - a^S_ij)^2 / (N * P)."""
    from oracle import pa_local_port as P
    g = torch.Generator().manual_seed(3)
    S = torch.randn(2, 4, 5, 7, generator=g, dtype=torch.float64)
    T = torch.randn(2, 6, 5, 7, generator=g, dtype=torch.float64)
    for k, d in ((3, 1), (5, 2), (3, 3)):
        fs, ft = P.normalise(S), P.normalise(T)
        r, total = (k - 1) // 2, 0.0
        for n, y, x, t, u in itertools.product(range(2), range(5), range(7), range(-r, r + 1), range(-r, r + 1)):
            yy, xx = y + t * d, x + u * d
            if 0 <= yy < 5 and 0 <= xx < 7:
                total += float((ft[n, :, y, x] * ft[n, :, yy, xx]).sum() - (fs[n, :, y, x] * fs[n, :, yy, xx]).sum()) ** 2
        assert float(P.local_affinity_loss(S, T, k, d)) == pytest.approx(total / (2 * _brute_pairs(5, 7, k, d)), rel=1e-12)


@pytest.mark.parametrize("k, d", [(3, 1), (5, 2), (3, 4)])
def test_gradcheck(k, d):
    """The restatement's autograd gradient (norm detached) against finite differences in float64, through the max pool: gradcheck of
    the loss with the student's pooled norms held at their values at S, which is the function whose exact gradient the detached norm
    defines."""
    import torch.nn.functional as F
    from oracle import pa_local_port as P
    g = torch.Generator().manual_seed(k * 10 + d)
    S = torch.randn(2, 3, 10, 12, generator=g, dtype=torch.float64, requires_grad=True)
    T = torch.randn(2, 4, 10, 12, generator=g, dtype=torch.float64)

    def pooled(x):
        return F.max_pool2d(x, (2, 2), (2, 2), 0, ceil_mode=True)
    rn = 1.0 / ((pooled(S.detach()) ** 2).sum(1, keepdim=True).sqrt() + 1e-8)
    ft = P.normalise(pooled(T))
    assert torch.autograd.gradcheck(lambda s: P.shifted_loss(pooled(s) * rn, ft, k, d), (S,), eps=1e-6, atol=1e-9)
    (want,) = torch.autograd.grad(P.pairwise_local_loss(S, T, 0.2, k, d), S)
    (got,) = torch.autograd.grad(P.shifted_loss(pooled(S) * rn, ft, k, d), S)
    assert float((got - want).norm()) <= 1e-12 * float(want.norm())


@pytest.fixture(scope="module")
def golden():
    from oracle import make_golden_pa_local as G
    return G.load()


def test_fixture_holds_every_case_and_student(golden):
    from oracle import make_golden_pa_local as G
    assert set(golden) == set(G.GOLDEN_CASES)
    assert {s["kind"] for s in G.GOLDEN_CASES.values()} == {"resnet18", "mobilenetv2", "espnet_c"}
    for name, spec in G.GOLDEN_CASES.items():
        pa = golden[name]["pa"]
        if isinstance(spec["window"], list):                         # a zero weight logs 0.0, the others a term
            assert len(pa) == len(spec["window"]) and all((v == 0.0) == (l == 0.0) for v, l in zip(pa, spec["cfg"]["lambda_pa"]))
        else:
            assert pa > 0.0


@pytest.mark.parametrize("name", ["r18_x1_local9d2_psp_global_96x128_b2", "espnet_c_psp_local15_360x480_b1"])
def test_fixture_reproduces_from_its_generator(golden, name):
    """The generator's step on the CPU reproduces the stored record (thread counts may reorder fp32 sums: 1e-4)."""
    from oracle import make_golden_pa_local as G
    gold, mine = golden[name], G.port_step(G.GOLDEN_CASES[name])
    for k in ("ce", "pi", "pa", "adv_g", "G", "D"):
        if k in gold:
            a, b = (mine[k], gold[k]) if isinstance(gold[k], list) else ([mine[k]], [gold[k]])
            assert a == pytest.approx(b, rel=1e-4, abs=1e-12), k
    assert torch.allclose(mine["logits_S"], gold["logits_S"], rtol=1e-3, atol=1e-4)
    for k, v in gold["student_grads"].items():
        assert mine["student_grads"][k]["norm"] == pytest.approx(v["norm"], rel=1e-3, abs=1e-9), k


@pytest.mark.parametrize("kw, match", [
    (dict(pa_window=9, lambda_pa=[0.5], pool_scale=[0.5]), "pa_window must be a list of 1 entries"),
    (dict(pa_window=[9], lambda_pa=0.5), "pa_window and pa_dilation must be scalars"),
    (dict(pa_window=9, pa_dilation=[1]), "pa_window and pa_dilation must be scalars"),
    (dict(pa_window=[9, None], pa_dilation=2, lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]), "pa_dilation must be a list of 2"),
    (dict(pa_window=[9], lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]), "lists must have 2 entries"),
    (dict(pa_window=[9, 9], pa_dilation=[1], lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]), "lists must have 2 entries"),
    (dict(pa_window=8), "pa_window must be None or an odd int in 3..15"),
    (dict(pa_window=1), "pa_window must be None or an odd int"),
    (dict(pa_window=17), "pa_window must be None or an odd int"),
    (dict(pa_window=True), "pa_window must be None or an odd int"),
    (dict(pa_window=9.0), "pa_window must be None or an odd int"),
    (dict(pa_window="9"), "pa_window must be None or an odd int"),
    (dict(pa_window=9, pa_dilation=0), "pa_dilation must be an int in 1..8"),
    (dict(pa_window=9, pa_dilation=9), "pa_dilation must be an int in 1..8"),
    (dict(pa_window=9, pa_dilation=True), "pa_dilation must be an int in 1..8"),
    (dict(pa_window=9, pa_dilation=2.0), "pa_dilation must be an int in 1..8"),
    (dict(pa_dilation=2), "pa_dilation 2 needs a local window"),
    (dict(pa_window=[None, 4], lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]), r"pair-wise level 1: pa_window must be None or an odd"),
    (dict(pa_window=[9, 19], lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]), r"pair-wise level 1: pa_window"),
    (dict(pa_window=[9, None], pa_dilation=[2, 2], lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]),
     r"pair-wise level 1: pa_dilation 2 needs a local window"),
    (dict(pa_window=[9, None], pa_dilation=[0, 1], lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.5]),
     r"pair-wise level 0: pa_dilation must be an int in 1..8"),
])
def test_netmodel_rejects_bad_windows_before_device_work(kw, match):
    """ValueError from NetModel's constructor naming the field (and the level in list form), before it looks for a device."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    with pytest.raises(ValueError, match=match):
        NetModel(make_args(**kw))


def test_valid_windows():
    import types
    from structure_knowledge_distillation_b200.utils.criterion import check_pa_windows
    lists = dict(lambda_pa=[0.5, 0.0, 0.5], pool_scale=[0.1, 0.5, 0.5])
    assert check_pa_windows(types.SimpleNamespace(pa_window=9, pa_dilation=2, lambda_pa=0.5)) == (9, 2)
    assert check_pa_windows(types.SimpleNamespace(pa_window=15, lambda_pa=0.5)) == (15, 1)
    assert check_pa_windows(types.SimpleNamespace(pa_window=[9, None, 3], pa_dilation=[2, 1, 8], **lists)) == [(9, 2), (None, 1), (3, 8)]
    assert check_pa_windows(types.SimpleNamespace(pa_window=[9, None, 3], **lists)) == [(9, 1), (None, 1), (3, 1)]
    assert check_pa_windows(types.SimpleNamespace(pa_window=(None, None, None), pa_dilation=(1, 1, 1), **lists)) == [(None, 1)] * 3
    assert check_pa_windows(types.SimpleNamespace(**lists)) is None
    assert check_pa_windows(types.SimpleNamespace(lambda_pa=0.5)) is None


def test_defaults_build_the_criteria_they_always_built():
    """make_args' defaults (pa_window None, pa_dilation 1): no window anywhere, and the criteria of the scalar and list forms are the
    fully connected ones they have always been."""
    from structure_knowledge_distillation_b200.utils.criterion import (CriterionPairWiseforWholeFeatAfterPool, CriterionPairWiseLocal,
                                                                        check_pa_levels, check_pa_windows, pair_wise_level_criteria)
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args()
    assert a.pa_window is None and a.pa_dilation == 1
    assert check_pa_windows(a) is None and check_pa_levels(a) is None
    b = make_args(lambda_pa=[0.5, 0.0, 1.0], pool_scale=[0.5, 0.5, 0.25])
    assert check_pa_windows(b) is None
    crits = pair_wise_level_criteria(check_pa_levels(b), check_pa_windows(b))
    assert [type(c) for c in crits] == [CriterionPairWiseforWholeFeatAfterPool] * 3
    assert [(c.feat_ind, c.scale) for c in crits] == [(-1, 0.5), (-2, 0.5), (-3, 0.25)]
    c = make_args(lambda_pa=[0.5, 0.5], pool_scale=[1 / 129, 0.5], pa_window=[9, None], pa_dilation=[2, 1])
    crits = pair_wise_level_criteria(check_pa_levels(c), check_pa_windows(c))
    assert [type(x) for x in crits] == [CriterionPairWiseLocal, CriterionPairWiseforWholeFeatAfterPool]
    assert (crits[0].feat_ind, crits[0].window, crits[0].dilation) == (-1, 9, 2)
