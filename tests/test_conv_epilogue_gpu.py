"""The wgmma convolution's fused epilogue, bit for bit: the same launch without an epilogue gives the raw fp32 accumulators, and
the fused result must equal float32 torch applying scale, shift, residual, activation and TF32 rounding to them one operation at a
time (each product and sum rounded on its own, never contracted into an FMA), on every tile mode and fragment edge."""
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [
    # N, Cin, H, W, Cout, k, stride, pad, dil, act
    (8, 256, 13, 21, 1024, 1, 1, 0, 1, "relu"),        # flat 1x1 GEMM, eight N tiles (teacher bottleneck conv3 class)
    (2, 64, 9, 13, 136, 1, 1, 0, 1, "relu"),           # ragged Cout: the last N tile holds 8 channels; last M tile partial
    (1, 128, 10, 11, 200, 3, 1, 2, 2, "leaky_relu"),   # im2col mode, dilation 2, ragged Cout
    (3, 64, 7, 9, 64, 3, 1, 1, 1, "relu"),             # BLOCK_N 64, tiles that wrap across images
    (2, 32, 9, 10, 30, 3, 1, 1, 1, "none"),            # BLOCK_N 32, odd-length last column pair
    (2, 64, 17, 15, 128, 3, 2, 1, 1, "relu"),          # stride 2
]


def _tf32_rn(t):
    """cvt.rn.tf32.f32 restated: round the 13 low mantissa bits away, to nearest, ties to even (finite values)."""
    b = t.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = ((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF) & 0xFFFFFFFF
    return torch.where(b >= 1 << 31, b - (1 << 32), b).to(torch.int32).view(torch.float32)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("im2col", [1, 0])
def test_epilogue_is_the_unfused_float32_sequence(case, im2col):
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    N, Cin, H, W, Cout, k, s, p, d, act = case
    g = torch.Generator(device="cuda").manual_seed(sum(case[:9]))
    x = ops.to_nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5)
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5
    sh = torch.randn(Cout, device="cuda", generator=g)
    oh, ow = ops.conv_out_hw(H, W, (k, k), s, p, d)
    # residual read through a channel slice of a wider buffer, output written into a channel slice of another
    res = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=Cout + 8)
    res.copy_(torch.randn(N, Cout, oh, ow, device="cuda", generator=g))
    try:
        lib().skd_set_conv_im2col(im2col)
        raw = ops.conv2d_fwd(x, w, s, p, d)
        for rnd in (False, True):
            ref = ((raw * sc[None, :, None, None]) + sh[None, :, None, None]) + res
            if act == "relu":
                ref = torch.relu(ref)
            elif act == "leaky_relu":
                ref = torch.where(ref < 0, ref * 0.1, ref)
            if rnd:
                ref = _tf32_rn(ref.contiguous())
            outs = []
            for _ in range(2):
                out = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=Cout + 20)
                ops.conv2d_fwd(x, w, s, p, d, scale=sc, shift=sh, residual=res, act=act, slope=0.1, out=out, round_tf32=rnd)
                outs.append(out)
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]), "run to run"
            assert torch.equal(outs[0], ref), (rnd, float((outs[0] - ref).abs().max()))
    finally:
        lib().skd_set_conv_im2col(1)


@pytest.mark.parametrize("M,Ncols,K", [(300, 136, 64), (1024, 1024, 96)])
def test_gemm_sum_of_squares_without_output(M, Ncols, K):
    """The affinity GEMM's reduction-only epilogue (no output tensor) sums every row of every tile, the first included."""
    from structure_knowledge_distillation_b200._cabi import lib
    g = torch.Generator(device="cuda").manual_seed(M + Ncols)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(Ncols, K, device="cuda", generator=g)
    D = torch.empty(M, Ncols, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    sums = torch.zeros(2, dtype=torch.float64, device="cuda")
    lib().skd_gemm_nt_sm100(M, Ncols, K, A.data_ptr(), K, B.data_ptr(), D.data_ptr(), Ncols, sums[0:1].data_ptr(), st)
    lib().skd_gemm_nt_sm100(M, Ncols, K, A.data_ptr(), K, B.data_ptr(), None, Ncols, sums[1:2].data_ptr(), st)
    torch.cuda.synchronize()
    ref = float((D.double() ** 2).sum())
    for s in sums.tolist():
        assert abs(s - ref) <= 1e-5 * ref, (s, ref)
