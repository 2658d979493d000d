"""The wgmma convolution's 256-row tiles compute what its 128-row tiles compute, bit for bit: every output element is the same k8
MMA sequence over the same TF32 operands followed by the same epilogue, only the tile that holds it differs.  Each launch runs with
skd_set_conv_tile_m(1) (always 128 rows), (2) (256 rows wherever the path can run) and (0) (the automatic choice), twice each."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = {
    # N, Cin, H, W, Cout, k, pad (= dil), dil
    "im2col_d1_P754": (2, 64, 13, 29, 128, 3, 1, 1),      # last tile: second 128-row box partly past P
    "im2col_d2_P600": (2, 96, 12, 25, 256, 3, 2, 2),      # last tile: second box wholly past P (not loaded)
    "im2col_d4_cout200": (1, 128, 17, 33, 200, 3, 4, 4),  # ragged Cout: the last N tile holds 72 channels
    "im2col_P99_cout512": (1, 64, 9, 11, 512, 3, 1, 1),   # P < 256: one partly filled tile per N tile
    "flat_cin2048": (1, 2048, 9, 37, 256, 1, 0, 1),       # flat 1x1 GEMM, P = 333
}
EPILOGUES = ["bn_relu", "bn_leaky_round", "residual_pitched", "residual_in_place"]


def _tf32_rn(t):
    """cvt.rn.tf32.f32 restated: round the 13 low mantissa bits away, to nearest, ties to even (finite values)."""
    b = t.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = ((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF) & 0xFFFFFFFF
    return torch.where(b >= 1 << 31, b - (1 << 32), b).to(torch.int32).view(torch.float32)


def _inputs(shape, seed):
    from structure_knowledge_distillation_b200 import ops
    N, Cin, H, W, Cout, k, p, d = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = ops.to_nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5)
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5
    sh = torch.randn(Cout, device="cuda", generator=g) * 0.1
    oh, ow = ops.conv_out_hw(H, W, (k, k), 1, p, d)
    r = torch.randn(N, Cout, oh, ow, device="cuda", generator=g)
    return x, w, sc, sh, r, oh, ow


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
def test_tile256_forward_bit_identical(name, epi):
    from structure_knowledge_distillation_b200 import ops
    shape = SHAPES[name]
    N, Cin, H, W, Cout, k, p, d = shape
    x, w, sc, sh, r, oh, ow = _inputs(shape, seed=sum(shape))
    res = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=Cout + 12)        # residual read through a channel slice of a wider buffer
    res.copy_(r)

    def run():
        if epi == "bn_relu":
            return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, act="relu")
        if epi == "bn_leaky_round":
            return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, act="leaky_relu", slope=0.1, round_tf32=True)
        if epi == "residual_pitched":
            out = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=Cout + 20)
            out.fill_(float("nan"))
            return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, residual=res, act="relu", out=out)
        out = ops.to_nhwc(r.clone())                                       # out = residual, as Bottleneck.frozen adds in place
        return ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, residual=out, act="relu", out=out)

    _assert_bit_identical(_per_mode(run))


def test_tile256_dgrad_with_residual_bit_identical():
    """The stride-1 data gradient (the forward kernel on dy with the flipped, transposed weights) plus a residual epilogue."""
    from structure_knowledge_distillation_b200 import ops
    N, Cin, H, W, Cout, k, p, d = 2, 256, 13, 21, 128, 3, 2, 2           # dx has 256 channels: two N tiles of 128, P = 546
    g = torch.Generator(device="cuda").manual_seed(7)
    dy = ops.to_nhwc(torch.randn(N, Cout, H, W, device="cuda", generator=g))
    w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5)
    res = ops.to_nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    _assert_bit_identical(_per_mode(lambda: ops.conv2d_dgrad(dy, w, (N, Cin, H, W), 1, p, d, residual=res)))


def test_tile256_against_float64():
    """Sanity of the 256-row path on its own: float64 convolution of the TF32-rounded operands, then the folded BN and ReLU."""
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    shape = SHAPES["im2col_d2_P600"]
    N, Cin, H, W, Cout, k, p, d = shape
    x, w, sc, sh, _, _, _ = _inputs(shape, seed=11)
    try:
        lib().skd_set_conv_tile_m(2)
        got = ops.conv2d_fwd(x, w, 1, p, d, scale=sc, shift=sh, act="relu").double()
    finally:
        lib().skd_set_conv_tile_m(0)
    w_oihw = w.permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(_tf32_rn(x.contiguous()).double(), _tf32_rn(w_oihw.contiguous()).double(), padding=p, dilation=d)
    ref = torch.relu(ref * sc.double()[None, :, None, None] + sh.double()[None, :, None, None])
    err = (got - ref).abs()
    assert float(err.max()) <= 1e-4 + 1e-4 * float(ref.abs().max()), float(err.max())
