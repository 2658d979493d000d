"""CPU checks of the full ESPNet student (ESPNet-C plus its decoder): the plain-torch oracle against tests/golden/espnet_full.pt.gz,
the parameter count and state-dict keys, restatements of the transposed convolution and of the resize adjoint the GPU kernels
compute, the size check, and loading an ESPNet-C checkpoint into `encoder.`."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cases, espnet_full_port, espnet_port, make_golden_espnet_full


def test_oracle_reproduces_fixture():
    gold = make_golden_espnet_full.load()
    name = "net_96x128_b2"
    got = make_golden_espnet_full.net_case(*make_golden_espnet_full.NET_CASES[name])
    for k in ("logits", "feat", "b1"):
        mine, ref = (got[k]["val"], gold[name][k]["val"]) if isinstance(got[k], dict) else cases.at_stored(got[k], gold[name][k])
        assert torch.allclose(mine, ref, rtol=1e-5, atol=1e-6), k
    assert abs(got["loss"] - gold[name]["loss"]) <= 1e-5 * abs(gold[name]["loss"])
    for pname, g in gold[name]["grads"].items():
        assert abs(got["grads"][pname]["norm"] - g["norm"]) <= 1e-4 * g["norm"] + 1e-8, pname


def test_parameter_count_keys_and_shapes():
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet
    ref = espnet_full_port.build_student(7)
    m = ESPNet(19, 2, 8)
    assert sum(p.numel() for p in ref.parameters()) == sum(p.numel() for p in m.parameters()) == 363462
    assert sum(p.numel() for p in m.encoder.parameters()) == 349193
    assert list(m.state_dict().keys()) == list(ref.state_dict().keys())
    for k in ("encoder.level1.conv.weight", "level3_C.conv.weight", "br.running_var", "up_l3.0.weight", "combine_l2_l3.0.act.weight",
              "combine_l2_l3.1.d16.conv.weight", "combine_l2_l3.1.bn.bn.weight", "up_l2.0.weight", "up_l2.1.act.weight",
              "conv.conv.weight", "classifier.weight"):
        assert k in m.state_dict(), k
    assert "br.weight" in m.state_dict() and not any(k.startswith("br.act") for k in m.state_dict())
    m.load_state_dict(ref.state_dict())
    ref.eval()
    with torch.no_grad():
        out = ref(torch.randn(1, 3, 96, 128))
    assert tuple(out[0].shape) == (1, 19, 96, 128) and out[1] is None and tuple(out[2].shape) == (1, 256, 12, 16)
    assert out[4].shape[1] == 131 and out[6].shape[1] == 19


def test_transposed_conv_as_gemm_and_depth_to_space():
    """functions.EspConvTranspose's forward: per output-row parity a, x (NHWC, Cin padded) times [b][co][ci] weights is a 1x1 GEMM
    to 2 * Coutp channels whose two halves are the output columns 2j and 2j + 1."""
    g = torch.Generator().manual_seed(0)
    for cin, cout, h, w in ((19, 19, 6, 7), (7, 5, 3, 4)):
        x = torch.randn(2, cin, h, w, generator=g, dtype=torch.float64)
        wt = torch.randn(cin, cout, 2, 2, generator=g, dtype=torch.float64)
        cin_p, cout_p = (cin + 3) // 4 * 4, (cout + 3) // 4 * 4
        wr = torch.zeros(2, 2, cout_p, cin_p, dtype=torch.float64)
        wr[:, :, :cout, :cin] = wt.permute(2, 3, 1, 0)
        wr = wr.reshape(2, 2 * cout_p, cin_p)
        xp = torch.zeros(2, h, w, cin_p, dtype=torch.float64)
        xp[..., :cin] = x.permute(0, 2, 3, 1)
        y = torch.zeros(2, 2 * h, 2 * w, cout_p, dtype=torch.float64)
        for a in range(2):
            gemm = xp @ wr[a].T                                             # (N, h, w, 2 * Coutp)
            y.view(2, h, 2, w, 2 * cout_p)[:, :, a] = gemm                  # rows 2i + a; columns 2j, 2j + 1 are consecutive
        ref = F.conv_transpose2d(x, wt, stride=2)
        assert torch.allclose(y.permute(0, 3, 1, 2)[:, :cout], ref, atol=1e-12)
        assert bool((y[..., cout:] == 0).all())
        # the data gradient is the 2x2 / stride-2 convolution of dy with w[ci][a][b][co]
        dy = torch.randn(2, cout, 2 * h, 2 * w, generator=g, dtype=torch.float64)
        xr = x.clone().requires_grad_(True)
        F.conv_transpose2d(xr, wt, stride=2).backward(dy)
        assert torch.allclose(F.conv2d(dy, wt, stride=2), xr.grad, atol=1e-12)


def _adj_weights(n_out, n_in):
    """(n_out, n_in) weights of espnet.cu's resample_adjoint_kernel along one axis, in its float32 arithmetic."""
    r = np.float32(np.float32(n_in - 1) / np.float32(n_out - 1)) if n_out > 1 else np.float32(0)
    m = np.zeros((n_out, n_in), dtype=np.float64)
    for o in range(n_out):
        f = np.float32(np.float32(o) * r)
        i0 = min(int(f), n_in - 1)
        i1 = min(i0 + 1, n_in - 1)
        lam = np.float32(f - np.float32(i0))
        m[o, i0] += np.float32(1) - lam
        m[o, i1] += lam
    return torch.from_numpy(m)


@pytest.mark.parametrize("src,dst", [((96, 128), (13, 17)), ((360, 480), (46, 61)), ((12, 16), (30, 41))])
def test_resize_adjoint_restatement_matches_autograd(src, dst):
    """The adjoint gather: d src[y][x] = sum over output pixels of wy(oy, y) * wx(ox, x) * d out[oy][ox] -- the transpose of the
    separable bilinear (align_corners=True) resize -- against autograd of F.interpolate."""
    g = torch.Generator().manual_seed(1)
    t = torch.randn(2, 3, *src, generator=g, dtype=torch.float64, requires_grad=True)
    dout = torch.randn(2, 3, *dst, generator=g, dtype=torch.float64)
    F.interpolate(t, size=dst, mode="bilinear", align_corners=True).backward(dout)
    ay, ax = _adj_weights(dst[0], src[0]), _adj_weights(dst[1], src[1])
    mine = torch.einsum("oy,ncop,px->ncyx", ay, dout, ax)
    # float32 source coordinates and weights, as the forward kernel's (o * r rounds to ~1e-5 of a pixel at 360 -> 46 rows)
    assert float((mine - t.grad).norm() / t.grad.norm()) < 1e-4


def test_sizes_not_multiple_of_8_raise():
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet
    for h, w in ((100, 128), (96, 130)):
        with pytest.raises(ValueError):
            ESPNet(19)(torch.zeros(1, 3, h, w))
        with pytest.raises(ValueError):
            espnet_full_port.ESPNet(19)(torch.zeros(1, 3, h, w))


def test_espnet_c_checkpoint_loads_into_encoder(tmp_path):
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    from structure_knowledge_distillation_b200.utils.utils import load_S_model
    enc = espnet_port.build_student(7)
    torch.save({"state_dict": enc.state_dict(), "step": 5, "epoch": 1, "best_mean_IU": 0.3}, tmp_path / "model_best.pth.tar")
    m = ESPNet(19)
    dec0 = {k: v.clone() for k, v in m.state_dict().items() if not k.startswith("encoder.")}
    assert load_S_model(make_args(S_resume=True, S_ckpt_path=str(tmp_path)), m, True) == "resume"
    for k, v in enc.state_dict().items():
        assert torch.equal(m.state_dict()["encoder." + k], v), k
    for k, v in dec0.items():
        assert torch.equal(m.state_dict()[k], v), k
    torch.save(enc.state_dict(), tmp_path / "imgnet.pth")
    m2 = ESPNet(19)
    assert load_S_model(make_args(is_student_load_imgnet=True, student_pretrain_model_imgnet=str(tmp_path / "imgnet.pth")), m2) == "imagenet"
    assert torch.equal(m2.state_dict()["encoder.level1.conv.weight"], enc.state_dict()["level1.conv.weight"])


def test_netmodel_arguments():
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    a = make_args(student="espnet")
    assert a.espnet_p == 2 and a.espnet_q == 8
    args = make_args(student="espnet", sync_bn=True)
    args.device = torch.device("cuda")
    with pytest.raises(ValueError):
        NetModel(args)
