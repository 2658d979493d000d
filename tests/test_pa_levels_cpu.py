"""Multi-level pair-wise distillation on the host: the float64-capable restatement of the reference's multi-level loop
(tools/pa_levels_oracle.py) against the golden the unmodified reference produced, NetModel's validation of list-valued
lambda_pa / pool_scale, and the level -> feature index order."""
import math
import types

import pytest
import torch


@pytest.fixture(scope="module")
def golden():
    from tools import pa_levels_oracle
    return pa_levels_oracle.load()


@pytest.mark.parametrize("name", ["levels5_pi_pa_96x128_b2", "level_x1_pi_pa_96x128_b2", "levels5_pi_pa_ho_wgangp_512_b1"])
def test_oracle_loop_reproduces_golden(golden, name):
    from tools import pa_levels_oracle as O
    gold = golden[name]
    rep = O.compare(O.port_step(O.GOLDEN_CASES[name]), gold)
    print("\nPARITY pa_levels oracle", name, {k: "%.1e" % v for k, v in rep.items()})
    assert all(v < 2e-4 for k, v in rep.items() if k != "student_grad_norm"), rep
    assert rep["student_grad_norm"] < 5e-3, rep
    lam = O.GOLDEN_CASES[name]["cfg"]["lambda_pa"]
    assert len(gold["pa"]) == len(lam)
    assert all((v == 0.0) == (l == 0.0) for v, l in zip(gold["pa"], lam))       # a zero weight logs 0.0, the others a term


def test_one_entry_list_selects_x1(golden):
    """Level 0 is preds[-1] (x1): the one-entry case's term is the five-level case's level-0 term (same seeds, same scale), not
    its PSP-feature term; the criteria NetModel builds read preds[-1] .. preds[-5] in level order."""
    from structure_knowledge_distillation_b200.utils.criterion import pair_wise_level_criteria
    one, five = golden["level_x1_pi_pa_96x128_b2"]["pa"], golden["levels5_pi_pa_96x128_b2"]["pa"]
    assert len(one) == 1 and one[0] == pytest.approx(five[0], rel=1e-6) and one[0] != pytest.approx(five[4], rel=1e-2)
    assert [c.feat_ind for c in pair_wise_level_criteria([(0.5, 0.5)])] == [-1]
    crits = pair_wise_level_criteria([(1.0, 0.5), (0.0, 0.25), (1.0, 0.125), (1.0, 1.0), (1.0, 0.3)])
    assert [c.feat_ind for c in crits] == [-1, -2, -3, -4, -5]
    assert [c.scale for c in crits] == [0.5, 0.25, 0.125, 1.0, 0.3]


def test_restated_levels_read_their_own_feature():
    """level_terms on synthetic 7-lists: level `ind` reads preds[-(ind + 1)] and nothing else."""
    from oracle import port
    from tools import pa_levels_oracle as O
    g = torch.Generator().manual_seed(0)
    S = [torch.randn(2, 8, 9, 12, generator=g, dtype=torch.float64) for _ in range(7)]
    T = [torch.randn(2, 16, 9, 12, generator=g, dtype=torch.float64) for _ in range(7)]
    total, terms = O.level_terms(S, T, [1.0, 0.0, 2.0], [0.5, 0.5, 0.25])
    assert terms[1] == 0.0
    assert float(terms[0]) == float(port.pairwise_loss(S[-1], T[-1], 0.5))
    assert float(terms[2]) == float(port.pairwise_loss(S[-3], T[-3], 0.25))
    assert float(total) == pytest.approx(float(terms[0]) + 2.0 * float(terms[2]), rel=1e-12)


@pytest.mark.parametrize("lam, scale, match", [
    ([0.5, 0.5], 0.5, "both be scalars or both be lists"),
    (0.5, [0.5], "both be scalars or both be lists"),
    ([0.5, 0.5], [0.5], "differ in length"),
    ([], [], "1..5 entries"),
    ([0.5] * 6, [0.5] * 6, "1..5 entries"),
    ([0.5, -0.1], [0.5, 0.5], "level 1: lambda_pa must be finite and >= 0"),
    ([math.inf], [0.5], "level 0: lambda_pa must be finite"),
    ([math.nan], [0.5], "level 0: lambda_pa must be finite"),
    ([0.5], [0.0], "level 0: pool_scale must be in"),
    ([0.5, 0.5], [0.5, 1.5], "level 1: pool_scale must be in"),
    ([0.5], [-0.5], "pool_scale must be in"),
    ([0.5], [math.nan], "pool_scale must be in"),
    ([0.5], ["x"], "must be numbers"),
])
def test_netmodel_rejects_bad_levels_before_device_work(lam, scale, match):
    """ValueError from NetModel's constructor, before it looks for a device (this runs without one)."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    with pytest.raises(ValueError, match=match):
        NetModel(make_args(lambda_pa=lam, pool_scale=scale))


def test_valid_levels_and_scalars():
    from structure_knowledge_distillation_b200.utils.criterion import check_pa_levels
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    assert check_pa_levels(make_args()) is None                                  # the defaults: the single term on preds[-5]
    assert check_pa_levels(make_args(lambda_pa=0.0, pool_scale=2.0)) is None     # scalars are taken as they always were
    assert check_pa_levels(make_args(lambda_pa=(1, 0.0), pool_scale=[1.0, 0.5])) == [(1.0, 1.0), (0.0, 0.5)]
    assert len(check_pa_levels(make_args(lambda_pa=[0.1] * 5, pool_scale=[0.5] * 5))) == 5


def test_print_info_prints_one_term_per_level(caplog):
    import logging
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.step_model import _LazyScalar
    groups = types.SimpleNamespace(param_groups=[{"lr": 0.01}])
    m = types.SimpleNamespace(G_solver=groups, D_solver=groups, G_loss=_LazyScalar(torch.tensor(3.0)), mc_G_loss=1.0, pi_G_loss=2.0,
                              pa_G_loss=[_LazyScalar(torch.tensor(0.25)), 0.0, _LazyScalar(torch.tensor(0.125))], D_loss=0.5)
    with caplog.at_level(logging.INFO):
        NetModel.print_info(m, 0, 7)
        m.pa_G_loss = 0.25
        NetModel.print_info(m, 0, 8)
    assert "pairwise:[0.25000, 0.00000, 0.12500])" in caplog.records[0].getMessage()
    assert "pairwise:0.25000)" in caplog.records[1].getMessage()
