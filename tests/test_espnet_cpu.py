"""CPU checks of the ESPNet-C student: the plain-torch oracle against tests/golden/espnet.pt.gz, the architecture's parameter count,
state-dict keys and output shapes, the package module's state dict against the oracle's, NetModel's arguments and refusals."""
import pytest
import torch

from oracle import cases, espnet_port, make_golden_espnet, port


def test_oracle_reproduces_fixture():
    gold = make_golden_espnet.load()
    name = "net_96x128_b2"
    b, h, w, train = make_golden_espnet.NET_CASES[name]
    got = make_golden_espnet.net_case(b, h, w, train)
    for k in ("logits", "feat", "b1"):
        mine, ref = cases.at_stored(got[k], gold[name][k]) if not isinstance(got[k], dict) else (got[k]["val"], gold[name][k]["val"])
        assert torch.allclose(mine, ref, rtol=1e-5, atol=1e-6), k
    assert abs(got["loss"] - gold[name]["loss"]) <= 1e-5 * abs(gold[name]["loss"])
    for pname, g in gold[name]["grads"].items():
        assert abs(got["grads"][pname]["norm"] - g["norm"]) <= 1e-4 * g["norm"] + 1e-8, pname


def test_parameter_count_keys_and_shapes():
    m = espnet_port.ESPNet_Encoder(19, 2, 8)
    assert sum(p.numel() for p in m.parameters()) == 349193
    keys = [k for k in m.state_dict() if not k.endswith("num_batches_tracked")]
    assert len(keys) == 154
    for k in ("level1.conv.weight", "level2_0.d16.conv.weight", "level2_0.act.weight", "level2.0.bn.bn.running_var", "b2.act.weight",
              "classifier.conv.weight"):
        assert k in keys, k
    m.eval()
    with torch.no_grad():
        for (h, w), (oh, ow) in (((360, 480), (45, 60)), ((512, 1024), (64, 128)), ((96, 128), (12, 16))):
            out = m(torch.randn(1, 3, h, w))
            assert tuple(out[0].shape) == (1, 19, oh, ow)
            assert out[1] is None and out[2].shape[1] == 256 and out[-1].shape[1] == 19 and out[4].shape[1] == 131


def test_package_module_state_dict_equals_oracle():
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet_C
    ref = espnet_port.build_student(7)
    m = ESPNet_C(19)
    a, b = m.state_dict(), ref.state_dict()
    assert list(a.keys()) == list(b.keys())
    for k in a:
        assert a[k].shape == b[k].shape, k
    m.load_state_dict(b)
    for k, v in m.state_dict().items():
        assert torch.equal(v, b[k]), k
    ref2 = espnet_port.ESPNet_Encoder(19)
    ref2.load_state_dict(m.state_dict())
    assert sum(p.numel() for p in m.parameters()) == 349193


def test_make_args_defaults():
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args()
    assert a.student == "resnet18" and a.espnet_p == 2 and a.espnet_q == 8
    assert make_args(student="espnet_c", espnet_q=3).espnet_q == 3


def test_value_errors():
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet_C
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    with pytest.raises(ValueError):
        ESPNet_C(19, 0, 8)
    with pytest.raises(ValueError):
        ESPNet_C(19, 2, 0)
    args = make_args(student="espnet_c", sync_bn=True)
    args.device = torch.device("cuda")
    with pytest.raises(ValueError):
        NetModel(args)
    with pytest.raises(ValueError):
        NetModel(make_args(student="mobilenet"))


def test_oracle_step_decisions():
    """Teacher tensors are resized only when the grids differ; the single-head CE equals the first term of the DSN loss."""
    preds_T = [torch.randn(1, 19, 46, 61), None, torch.randn(1, 8, 46, 61), None, None, None, None]
    out = espnet_port.resample_teacher(preds_T, (45, 60))
    assert out[0].shape[2:] == (45, 60) and out[2].shape[2:] == (45, 60)
    assert espnet_port.resample_teacher(preds_T, (46, 61)) is preds_T
    images, labels = port.synthetic_batch(1, 64, 96, seed=0)
    logits = torch.randn(1, 19, 8, 12)
    ce = espnet_port.ce_loss([logits], labels)
    both = port.dsn_ce_loss([logits, torch.zeros_like(logits)], labels)
    assert abs(float(both) - float(ce) - 0.4 * float(torch.log(torch.tensor(19.0)))) < 1e-4
