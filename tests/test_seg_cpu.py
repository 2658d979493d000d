"""SegModel's host side without a GPU: oracle/port.py's training-mode PSPNet-ResNet101 against the reference's steps in
tests/golden/seg_steps.pt.gz (oracle/make_golden_seg.py), the `seg_model` choices, ImageNet initialisation by key intersection, and the
checkpoint contract: what SegModel saves loads through load_T_model as NetModel's teacher."""
import argparse
import logging

import pytest
import torch


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_port_matches_reference_golden():
    """Two SGD steps of the port's PSPNet-ResNet101 (19 classes, CriterionDSN) equal the reference's: loss, logits, every gradient norm
    and the sampled parameters after each step."""
    from oracle import make_golden_seg as G, port
    gold = G.load()["r101_c19"]["steps"]
    mine = G.port_case("r101_c19")
    assert len(mine) == len(gold) == G.STEPS
    for a, b in zip(mine, gold):
        assert abs(a["loss"] - b["loss"]) / abs(b["loss"]) < 1e-5, (a["loss"], b["loss"])
        assert _rel(a["logits"], b["logits"]) < 1e-4
        worst = max(abs(a["grads"][k]["norm"] - v["norm"]) / v["norm"] for k, v in b["grads"].items() if v["norm"] > 1e-6)
        assert worst < 1e-3, worst
        for k, v in b["params"].items():
            assert torch.allclose(a["params"][k], v, rtol=1e-5, atol=1e-7), k
    assert port.PSPNet.CONFIGS["resnet101"][1] == (3, 4, 23, 3)


def test_golden_covers_the_cases():
    from oracle import make_golden_seg as G
    gold = G.load()
    assert set(gold) == set(G.CASES)
    for name, (arch, classes, ohem) in G.CASES.items():
        steps = gold[name]["steps"]
        assert len(steps) == G.STEPS and steps[0]["logits"].shape[1] == classes
        if ohem:                                       # OHEM keeps a strict subset of the valid pixels
            assert all(0 < k < gold[name]["valid"] for k in gold[name]["kept"])


def _args(**kw):
    d = dict(classes_num=19, lr_g=1e-2, momentum=0.9, weight_decay=5e-4, num_steps=100, power=0.9, device=torch.device("cuda"))
    d.update(kw)
    return argparse.Namespace(**d)


@pytest.mark.parametrize("kw,msg", [
    (dict(seg_model="resnet50"), "seg_model"),
    (dict(seg_model=""), "seg_model"),
    (dict(classes_num=33), "classes_num"),
    (dict(classes_num=0), "classes_num"),
    (dict(seg_model="espnet", sync_bn=True), "sync_bn"),
    (dict(seg_model="espnet_c", sync_bn=True), "sync_bn"),
    (dict(seg_model="mobilenetv2", sync_bn=True), "sync_bn"),
])
def test_seg_model_validation(kw, msg):
    """Unknown networks, class counts outside 1..32 and sync_bn with a per-rank-statistics network raise before any device work."""
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    with pytest.raises(ValueError, match=msg):
        SegModel(_args(**kw))


def test_seg_network_kinds():
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Bottleneck
    from structure_knowledge_distillation_b200.networks.step_model import SEG_MODELS, build_seg_network
    assert SEG_MODELS[0] == "resnet101"
    r101 = build_seg_network("resnet101", 21)
    assert isinstance(r101.layer3[0], Bottleneck) and len(r101.layer3) == 23 and r101.head.out_channels == 21
    assert isinstance(build_seg_network("resnet18", 19).layer1[0], BasicBlock)
    for kind in ("espnet_c", "espnet", "mobilenetv2"):
        assert build_seg_network(kind, 19) is not None
    with pytest.raises(ValueError):
        build_seg_network("vgg16", 19)


def test_precision_policies():
    """The policies set exactly the convolutions they name, and SegModel's choice leaves the ResNet constructor's flags alone (NetModel's
    student and teacher keep them)."""
    from structure_knowledge_distillation_b200.networks.pspnet_combine import Conv2d
    from structure_knowledge_distillation_b200.networks.seg_model import DEFAULT_PRECISION, set_precision_policy
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    net = build_seg_network("resnet101", 19)
    fresh = {n: m.precise for n, m in net.named_modules() if isinstance(m, Conv2d)}
    early = {n for n, p in fresh.items() if p}
    assert early and all(n.startswith(("conv", "layer1.", "layer2.")) for n in early)
    set_precision_policy(net, "early")
    assert {n for n, m in net.named_modules() if isinstance(m, Conv2d) and m.precise} == early
    set_precision_policy(net, "layer3")
    on = {n for n, m in net.named_modules() if isinstance(m, Conv2d) and m.precise}
    assert on == early | {n for n in fresh if n.startswith("layer3.")}
    set_precision_policy(net, "all")
    assert all(m.precise for m in net.modules() if isinstance(m, Conv2d))
    with pytest.raises(ValueError):
        set_precision_policy(net, "fp64")
    assert set(DEFAULT_PRECISION) == {"resnet101", "resnet18"}
    assert {n for n, m in build_seg_network("resnet101", 19).named_modules() if isinstance(m, Conv2d) and m.precise} == early


def _imagenet_state(net, seed=0):
    """A deep-stem ImageNet ResNet-101 checkpoint as such checkpoints come: the backbone (conv1-3, bn1-3, layer1-4) plus the
    classifier `fc` and BN sample counters the segmentation network does not have."""
    g = torch.Generator().manual_seed(seed)
    sd = {k: torch.randn(v.shape, generator=g) for k, v in net.state_dict().items()
          if k.split(".")[0] in ("conv1", "conv2", "conv3", "bn1", "bn2", "bn3", "layer1", "layer2", "layer3", "layer4")}
    sd["fc.weight"] = torch.randn(1000, 2048, generator=g)
    sd["fc.bias"] = torch.randn(1000, generator=g)
    sd["bn1.num_batches_tracked"] = torch.tensor(7)
    return sd


def test_imagenet_init_loads_by_intersection(tmp_path, caplog):
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    from structure_knowledge_distillation_b200.utils.utils import load_seg_model
    net = build_seg_network("resnet101", 19)
    sd = _imagenet_state(net)
    path = tmp_path / "resnet101-imagenet.pth"
    torch.save(sd, path)
    before = {k: v.clone() for k, v in net.state_dict().items()}
    with caplog.at_level(logging.INFO):
        assert load_seg_model(_args(is_load_imgnet=True, pretrain_model_imgnet=str(path)), net) == "imagenet"
    after = net.state_dict()
    n = 0
    for k, v in after.items():
        if k in sd:
            assert torch.equal(v, sd[k]), k
            n += 1
        else:
            assert k.startswith(("pspmodule.", "head.", "dsn.")) and torch.equal(v, before[k]), k
    assert n == len(sd) - 3
    assert any(("%d of %d tensors" % (n, len(sd))) in r.getMessage() for r in caplog.records), [r.getMessage() for r in caplog.records]


def test_resume_restores_state_and_last_step(tmp_path):
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    from structure_knowledge_distillation_b200.utils.utils import load_seg_model
    src = build_seg_network("resnet18", 19)
    torch.save(dict(state_dict={"module." + k: v for k, v in src.state_dict().items()}, step=1234, epoch=3, best_mean_IU=0.5),
               tmp_path / "model_best.pth.tar")
    args = _args(resume=True, ckpt_path=str(tmp_path))
    dst = build_seg_network("resnet18", 19)
    assert load_seg_model(args, dst, False) == "resume"
    assert args.last_step == 1234 and args.start_epoch == 3 and args.best_mean_IU == 0.5
    assert all(torch.equal(a, b) for a, b in zip(src.state_dict().values(), dst.state_dict().values()))


def test_saved_state_dict_loads_as_netmodel_teacher(tmp_path):
    """A SegModel checkpoint (model.state_dict() of Res_pspnet(Bottleneck, [3, 4, 23, 3])) goes through load_T_model, whose
    `head.0.` / `head.1.` remap leaves its keys untouched, into a freshly built teacher with every key matched."""
    from structure_knowledge_distillation_b200.networks.pspnet_combine import Bottleneck, Res_pspnet
    from structure_knowledge_distillation_b200.utils.utils import load_T_model
    torch.manual_seed(1)
    src = Res_pspnet(Bottleneck, [3, 4, 23, 3], num_classes=21)
    with torch.no_grad():
        for b in src.buffers():
            b.uniform_(0.5, 1.5)
    sd = src.state_dict()
    assert not any(k.startswith(("head.0.", "head.1.", "fc.")) for k in sd)
    path = tmp_path / "CS_scenes_100_0.5.pth"
    torch.save(sd, path)
    torch.manual_seed(2)
    teacher = Res_pspnet(Bottleneck, [3, 4, 23, 3], num_classes=21)
    assert load_T_model(teacher, str(path)) is True                 # load_state_dict(strict=True) inside: no key missing or unexpected
    got = teacher.state_dict()
    assert set(got) == set(sd)
    assert all(torch.equal(got[k], v) for k, v in sd.items())
