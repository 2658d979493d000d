"""Short K loops on the wgmma convolution's 256-row tiles: the same bit-for-bit check as test_conv_tile256_gpu.py for the short-K
launches the tile selection sends to 256 rows (K = 18 .. 72 steps, and a flat 1x1 with K = 32 and 16 N tiles).  Each launch runs with
skd_set_conv_tile_m(1) (always 128 rows), (2) (256 rows wherever the path can run) and (0) (the automatic choice), twice each, and
every output must equal the 128-row output bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = {
    # N, Cin, H, W, Cout, k, pad (= dil), dil
    "flat_k32_16ntiles": (1, 1024, 11, 43, 2048, 1, 0, 1),   # flat 1x1 GEMM, K = 32, 16 N tiles, P = 473
    "im2col_cin64_k18": (2, 64, 19, 27, 256, 3, 1, 1),       # 3x3 with Cin 64: K = 9 x 2 = 18
    "im2col_d2_k72": (2, 256, 13, 23, 256, 3, 2, 2),         # 3x3 d2 256->256, layer3's K = 72
    "im2col_cin64_k18_one_ntile": (1, 64, 23, 31, 128, 3, 1, 1),   # the stem's 64->128: a lone N tile
}
EPILOGUES = ["bn_relu", "bn_leaky_round", "none_elu", "residual_pitched", "residual_in_place"]


def _per_mode(fn):
    """fn() -> output tensor; run twice under each tile mode -> {mode: [out, out]}"""
    from structure_knowledge_distillation_b200._cabi import lib
    outs = {}
    try:
        for mode in (1, 2, 0):
            lib().skd_set_conv_tile_m(mode)
            outs[mode] = [fn().clone() for _ in range(2)]
    finally:
        lib().skd_set_conv_tile_m(0)
    torch.cuda.synchronize()
    return outs


def _assert_bit_identical(outs):
    ref = outs[1][0]
    for mode, (a, b) in outs.items():
        assert torch.equal(a, b), ("run to run", mode)
        assert torch.equal(a, ref), (mode, float((a - ref).abs().max()))


@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("name", list(SHAPES))
def test_tile256_short_k_forward_bit_identical(name, epi):
    from structure_knowledge_distillation_b200 import ops
    N, Cin, H, W, Cout, k, p, d = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(sum(SHAPES[name]))
    x = ops.to_nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5)
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5
    sh = torch.randn(Cout, device="cuda", generator=g) * 0.1
    oh, ow = ops.conv_out_hw(H, W, (k, k), 1, p, d)
    r = torch.randn(N, Cout, oh, ow, device="cuda", generator=g)
    res = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=Cout + 12)        # residual read through a channel slice of a wider buffer
    res.copy_(r)

    def run():
        if epi == "bn_relu":
            return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, act="relu")
        if epi == "bn_leaky_round":
            return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, act="leaky_relu", slope=0.1, round_tf32=True)
        if epi == "none_elu":
            return ops.conv2d_fwd(x, w, 1, p, d, act="elu")
        if epi == "residual_pitched":
            out = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=Cout + 20)
            out.fill_(float("nan"))
            return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, residual=res, act="relu", out=out)
        out = ops.to_nhwc(r.clone())                                       # out = residual, as Bottleneck.frozen adds in place
        return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, residual=out, act="relu", out=out)

    _assert_bit_identical(_per_mode(run))


@pytest.mark.parametrize("Cin,Cout,k,p,d", [(256, 256, 3, 2, 2), (128, 256, 3, 2, 2), (256, 64, 3, 1, 1), (512, 1024, 1, 0, 1)])
def test_tile256_short_k_dgrad_bit_identical(Cin, Cout, k, p, d):
    """The stride-1 data gradient (the forward kernel on dy with the flipped, transposed weights): K = 72 (layer3's 3x3 d2 256->256
    and 128->256), 18 (64 dy channels) and 32 (a 1x1 with 1024 dy channels), plus a residual epilogue."""
    from structure_knowledge_distillation_b200 import ops
    N, H, W = 2, 13, 21
    g = torch.Generator(device="cuda").manual_seed(Cin + Cout + k)
    dy = ops.to_nhwc(torch.randn(N, Cout, H, W, device="cuda", generator=g))
    w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5)
    res = ops.to_nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    _assert_bit_identical(_per_mode(lambda: ops.conv2d_dgrad(dy, w, (N, Cin, H, W), 1, p, d)))
    _assert_bit_identical(_per_mode(lambda: ops.conv2d_dgrad(dy, w, (N, Cin, H, W), 1, p, d, residual=res)))
