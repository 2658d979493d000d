"""CPU checks of the MobileNetV2 student: the plain-torch oracle against tests/golden/mobilenet.pt.gz, the package module's state dict
against the oracle's, the backbone against torchvision's mobilenet_v2 (when torchvision is importable), ImageNet initialisation through
load_S_model, NetModel's arguments and refusals."""
import pytest
import torch

from oracle import cases, make_golden_mobilenet, mobilenet_port


def test_oracle_reproduces_fixture():
    gold = make_golden_mobilenet.load()
    name = "net_96x128_b2"
    b, h, w, train = make_golden_mobilenet.NET_CASES[name]
    got = make_golden_mobilenet.net_case(b, h, w, train)
    for k in ("logits", "dsn", "feat", "f3"):
        mine, ref = cases.at_stored(got[k], gold[name][k]) if not isinstance(got[k], dict) else (got[k]["val"], gold[name][k]["val"])
        assert torch.allclose(mine, ref, rtol=1e-5, atol=1e-6), k
    assert abs(got["loss"] - gold[name]["loss"]) <= 1e-5 * abs(gold[name]["loss"])
    for k, v in gold[name]["running"].items():
        assert torch.allclose(got["running"][k], v, rtol=1e-5, atol=1e-6), k
    for pname, g in gold[name]["grads"].items():
        assert abs(got["grads"][pname]["norm"] - g["norm"]) <= 1e-4 * g["norm"] + 1e-8, pname


def test_parameter_count_and_output_shapes():
    m = mobilenet_port.MobileNetV2Student(19)
    assert sum(p.numel() for p in m.parameters()) == 3051174
    assert sum(p.numel() for p in m.features.parameters()) == 1811712
    m.eval()
    with torch.no_grad():
        for (h, w), (oh, ow) in (((360, 480), (45, 60)), ((512, 1024), (64, 128)), ((96, 128), (12, 16))):
            out = m(torch.randn(1, 3, h, w))
            assert [tuple(t.shape[1:]) for t in out] == [(19, oh, ow), (19, oh, ow), (128, oh, ow), (320, oh, ow), (96, oh, ow),
                                                           (32, oh, ow), (24, 2 * oh, 2 * ow)]


def test_package_module_state_dict_equals_oracle():
    from structure_knowledge_distillation_b200.networks.mobilenet import MobileNetV2
    ref = mobilenet_port.build_student(7)
    m = MobileNetV2(19)
    a, b = m.state_dict(), ref.state_dict()
    assert list(a.keys()) == list(b.keys())
    for k in a:
        assert a[k].shape == b[k].shape, k
    m.load_state_dict(b)
    for k, v in m.state_dict().items():
        assert torch.equal(v, b[k]), k
    assert m.features[4].conv[1][0].weight.shape == (144, 1, 3, 3)
    assert "features.4.conv.1.0.weight" in a and "features.4.conv.1.1.running_var" in a and "pspmodule.bottleneck.1.weight" in a


def test_depthwise_geometry_follows_the_dilation_rule():
    from structure_knowledge_distillation_b200.networks.mobilenet import MobileNetV2
    m = MobileNetV2(19)
    got = {}
    for i in range(1, 18):
        dw = m.features[i].conv[-3][0]
        got[i] = (dw.stride, dw.dilation)
    assert got[2] == got[4] == (2, 1)
    assert all(got[i] == (1, 1) for i in (1, 3, 5, 6, 7))
    assert all(got[i] == (1, 2) for i in range(8, 15))
    assert all(got[i] == (1, 4) for i in (15, 16, 17))
    assert [i for i in range(1, 18) if m.features[i].use_res_connect] == [3, 5, 6, 8, 9, 10, 12, 13, 15, 16]


def _torchvision():
    return pytest.importorskip("torchvision")


def test_backbone_keys_and_shapes_equal_torchvision():
    tv = _torchvision().models.mobilenet_v2().state_dict()
    want = {k: v.shape for k, v in tv.items() if k.startswith("features.") and int(k.split(".")[1]) <= 17}
    got = {k: v.shape for k, v in mobilenet_port.MobileNetV2Student(19).state_dict().items() if k.startswith("features.")}
    assert list(got) == list(want)
    assert got == want


def test_oracle_backbone_equals_dilated_torchvision():
    tvm = _torchvision().models.mobilenet_v2()
    ref = mobilenet_port.build_student(3)
    tvm.load_state_dict({**tvm.state_dict(), **{k: v for k, v in ref.state_dict().items() if k.startswith("features.")}})
    mobilenet_port.dilate_torchvision(tvm)
    x = torch.randn(2, 3, 96, 128, generator=torch.Generator().manual_seed(0))
    for train in (False, True):
        tvm.train(train); ref.train(train)
        with torch.no_grad():
            want = tvm.features[:18](x)
            got = ref.features(x)
        assert got.shape == want.shape == (2, 320, 12, 16)
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), float((got - want).abs().max())


def test_torchvision_state_dict_loads_through_load_S_model(tmp_path):
    from structure_knowledge_distillation_b200.networks.mobilenet import MobileNetV2
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    from structure_knowledge_distillation_b200.utils.utils import load_S_model
    torch.manual_seed(1)
    tv = mobilenet_port.MobileNetV2Student(19).state_dict()
    tv = {k: v for k, v in tv.items() if k.startswith("features.")}
    tv["features.18.0.weight"] = torch.randn(1280, 320, 1, 1)           # torchvision's last layer and classifier: not ours
    tv["classifier.1.weight"] = torch.randn(1000, 1280)
    path = tmp_path / "mobilenet_v2_imagenet.pth"
    torch.save(tv, path)
    torch.manual_seed(2)
    m = MobileNetV2(19)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    args = make_args(student="mobilenetv2", is_student_load_imgnet=True, student_pretrain_model_imgnet=str(path), S_ckpt_path="")
    assert load_S_model(args, m, False) == "imagenet"
    sd = m.state_dict()
    n = 0
    for k, v in sd.items():
        if k.startswith("features."):
            assert torch.equal(v, tv[k]), k
            n += 1
        else:
            assert torch.equal(v, before[k]), k
    assert n == len([k for k in tv if k.startswith("features.") and int(k.split(".")[1]) <= 17])


def test_make_args_accepts_mobilenetv2():
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args(student="mobilenetv2")
    assert a.student == "mobilenetv2" and make_args().student == "resnet18"


def test_value_errors():
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.mobilenet import DepthwiseConv
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    args = make_args(student="mobilenetv2", sync_bn=True)
    args.device = torch.device("cuda")
    with pytest.raises(ValueError, match="sync_bn"):
        NetModel(args)
    with pytest.raises(ValueError, match="mobilenetv2"):
        NetModel(make_args(student="mobilenet_v3"))
    x = torch.zeros(1, 8, 5, 5)
    for c, wshape, stride, dil in ((6, (6, 1, 3, 3), 1, 1), (8, (8, 1, 5, 5), 1, 1), (8, (8, 1, 3, 3), 3, 1), (8, (8, 1, 3, 3), 1, 0),
                                   (8, (8, 8, 3, 3), 1, 1)):
        with pytest.raises(ValueError):
            ops.dwconv3x3_fwd(torch.zeros(1, c, 5, 5), torch.zeros(wshape), stride, dil)
    with pytest.raises(ValueError):
        ops.dwconv3x3_dgrad(x, torch.zeros(8, 1, 3, 3), (1, 8, 5, 5), 2, 0)
    with pytest.raises(ValueError):
        ops.dwconv3x3_wgrad(torch.zeros(1, 12 + 2, 5, 5), x, 1, 1)
    with pytest.raises(ValueError):
        DepthwiseConv(20, 4, 1)
