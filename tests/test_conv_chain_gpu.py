"""The chained frozen-bottleneck launch (skd_conv1x1_chain_sm100: block i's conv3 and block i+1's conv1 in one kernel) computes both
outputs bit for bit as the two unfused wgmma launches do, at every layer1-3 pair shape of the benchmark, on ragged and batch-1 pixel
counts, with the output written over the residual, and through the whole teacher forward, eagerly and under CUDA-graph replay."""
import pytest
import torch

pytestmark = pytest.mark.gpu

PAIRS = {
    # N, planes (conv3 Cin, conv1 Cout), H, W: conv3 planes -> 4 * planes, then conv1 4 * planes -> planes
    "layer1_b8": (8, 64, 129, 257),
    "layer2_b8": (8, 128, 65, 129),
    "layer3_b8": (8, 256, 65, 129),
    "layer3_b1_P117": (1, 256, 9, 13),        # one partly filled tile, its second 64-row half partly past P
    "layer1_b1_P143": (1, 64, 11, 13),        # second tile: 15 pixels, its second half wholly past P
    "layer2_b1_P187": (1, 128, 11, 17),
}


def _operands(N, planes, H, W, seed):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    c3 = 4 * planes
    x3 = ops.to_nhwc(torch.relu(torch.randn(N, planes, H, W, device="cuda", generator=g)))
    res = ops.to_nhwc(torch.randn(N, c3, H, W, device="cuda", generator=g))
    w3 = ops.weight_ohwi(torch.randn(c3, planes, 1, 1, device="cuda", generator=g) / planes ** 0.5)
    w1 = ops.weight_ohwi(torch.randn(planes, c3, 1, 1, device="cuda", generator=g) / c3 ** 0.5)
    bn = [(torch.rand(c, device="cuda", generator=g) + 0.5, torch.randn(c, device="cuda", generator=g) * 0.1) for c in (c3, planes)]
    return x3, res, w3, w1, bn[0], bn[1]


def _unfused(x3, res, w3, w1, bn3, bn1):
    from structure_knowledge_distillation_b200 import ops
    y3 = ops.conv2d_fwd(x3, w3, 1, 0, 1, scale=bn3[0], shift=bn3[1], residual=res, act="relu")
    y1 = ops.conv2d_fwd(y3, w1, 1, 0, 1, scale=bn1[0], shift=bn1[1], act="relu")
    return y3, y1


@pytest.mark.parametrize("name", list(PAIRS))
def test_chain_equals_the_two_launches(name):
    from structure_knowledge_distillation_b200 import ops
    x3, res, w3, w1, bn3, bn1 = _operands(*PAIRS[name], seed=sum(PAIRS[name]))
    ref3, ref1 = _unfused(x3, res, w3, w1, bn3, bn1)
    outs = [ops.conv1x1_chain(x3, w3, *bn3, res, w1, *bn1) for _ in range(2)]
    torch.cuda.synchronize()
    for y3, y1 in outs:
        assert torch.equal(y3, ref3), float((y3 - ref3).abs().max())
        assert torch.equal(y1, ref1), float((y1 - ref1).abs().max())


@pytest.mark.parametrize("name", ["layer3_b1_P117", "layer2_b8"])
def test_chain_in_place_residual(name):
    """y3 written over the residual it reads."""
    from structure_knowledge_distillation_b200 import ops
    x3, res, w3, w1, bn3, bn1 = _operands(*PAIRS[name], seed=7)
    ref3, ref1 = _unfused(x3, res, w3, w1, bn3, bn1)
    buf = res.clone(memory_format=torch.channels_last)
    y3, y1 = ops.conv1x1_chain(x3, w3, *bn3, buf, w1, *bn1, out3=buf)
    torch.cuda.synchronize()
    assert y3.data_ptr() == buf.data_ptr()
    assert torch.equal(buf, ref3), float((buf - ref3).abs().max())
    assert torch.equal(y1, ref1), float((y1 - ref1).abs().max())


def _teacher():
    from structure_knowledge_distillation_b200.networks.pspnet_combine import Bottleneck, Res_pspnet
    torch.manual_seed(0)
    net = Res_pspnet(Bottleneck, [3, 4, 23, 3], 19).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    for m in net.modules():
        if hasattr(m, "running_var"):
            m.running_mean.copy_(torch.randn(m.running_mean.shape, device="cuda", generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.running_var.shape, device="cuda", generator=g) + 0.5)
    for p in net.parameters():
        p.requires_grad_(False)
    return net


def test_teacher_forward_chained_equals_unchained_eager_and_graph():
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    net = _teacher()
    img = torch.randn(2, 3, 97, 161, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    log = []
    try:
        with torch.no_grad():
            lib().skd_set_conv_chain(1)
            ref = [t.clone() for t in net(img)]
            lib().skd_set_conv_chain(0)
            ops.CONV_EVENT_LOG = log
            eager = [t.clone() for t in net(img)]
            ops.CONV_EVENT_LOG = None
            calls = [r[3] for r in log if isinstance(r[3][-1], str) and r[3][-1].startswith("chain1x1")]
            stream = torch.cuda.Stream()
            stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(stream):
                net(img)                                             # warm-up on the capture stream
            torch.cuda.current_stream().wait_stream(stream)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static = net(img)
            graph.replay()
            torch.cuda.synchronize()
            replayed = [t.clone() for t in static]
    finally:
        ops.CONV_EVENT_LOG = None
        lib().skd_set_conv_chain(0)
    assert len(calls) == 2 + 3 + 22, calls                            # every layer1-3 pair chained, nothing in layer4
    for i, (r, e, g) in enumerate(zip(ref, eager, replayed)):
        assert torch.equal(e, r), (i, float((e - r).abs().max()))
        assert torch.equal(g, r), (i, float((g - r).abs().max()))
