"""The wgmma convolution's TMA epilogue (short-K flat / im2col launches with a residual: residual loaded and output stored through a
shared-memory tile), bit for bit against float32 torch applying scale, shift, residual, activation and TF32 rounding to the raw accumulators one
operation at a time, and bit for bit run to run."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = -12345.5


def _tf32_rn(t):
    """cvt.rn.tf32.f32 restated: round the 13 low mantissa bits away, to nearest, ties to even (finite values)."""
    b = t.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = ((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF) & 0xFFFFFFFF
    return torch.where(b >= 1 << 31, b - (1 << 32), b).to(torch.int32).view(torch.float32)


def _operands(N, Cin, H, W, Cout, k, seed):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = ops.to_nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5)
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5
    sh = torch.randn(Cout, device="cuda", generator=g)
    return x, w, sc, sh, g


def _reference(raw, sc, sh, res, act, rnd):
    ref = (raw * sc[None, :, None, None]) + sh[None, :, None, None]
    if res is not None:
        ref = ref + res
    if act == "relu":
        ref = torch.relu(ref)
    elif act == "leaky_relu":
        ref = torch.where(ref < 0, ref * 0.1, ref)
    return _tf32_rn(ref.contiguous()) if rnd else ref


def _sliced_out(N, Cout, oh, ow, pitch, c_off, extra_rows):
    """(N, Cout, oh, ow) NHWC view at channel c_off of a sentinel-filled buffer of pitch `pitch` with `extra_rows` pixels past the end."""
    buf = torch.full(((N * oh * ow + extra_rows) * pitch,), SENTINEL, device="cuda")
    view = buf.as_strided((N, Cout, oh, ow), (oh * ow * pitch, 1, ow * pitch, pitch), c_off)
    return buf, view


CASES = [
    # N, Cin, H, W, Cout, k, stride, pad, dil, act, out pitch
    (8, 256, 65, 129, 1024, 1, 1, 0, 1, "relu", None),        # teacher layer3 conv3 at the benchmark size: ~32 tiles per CTA
    (2, 64, 9, 13, 136, 1, 1, 0, 1, "relu", None),            # last M tile partly filled (234 pixels), last N tile 8 channels
    (1, 32, 10, 11, 200, 3, 1, 2, 2, "leaky_relu", None),     # im2col mode, dilation 2, ragged Cout
    (3, 32, 7, 9, 64, 3, 1, 1, 1, "none", None),              # BLOCK_N 64, tiles that wrap across images
    (2, 32, 9, 10, 30, 1, 1, 0, 1, "relu", None),             # BLOCK_N 32, odd-length last column pair
    (2, 64, 9, 13, 136, 1, 1, 0, 1, "relu", 138),             # pitch not a whole float4: the register epilogue, still exact
]


@pytest.mark.parametrize("case", CASES)
def test_tma_epilogue_is_the_unfused_float32_sequence(case):
    from structure_knowledge_distillation_b200 import ops
    N, Cin, H, W, Cout, k, s, p, d, act, opitch = case
    x, w, sc, sh, g = _operands(N, Cin, H, W, Cout, k, sum(case[:9]))
    oh, ow = ops.conv_out_hw(H, W, (k, k), s, p, d)
    res = ops.to_nhwc(torch.randn(N, Cout, oh, ow, device="cuda", generator=g))
    raw = ops.conv2d_fwd(x, w, s, p, d)
    for rnd in (False, True):
        ref = _reference(raw, sc, sh, res, act, rnd)
        outs = []
        for _ in range(2):
            out = ops.empty_nhwc(N, Cout, oh, ow, "cuda", pitch=opitch)
            ops.conv2d_fwd(x, w, s, p, d, scale=sc, shift=sh, residual=res, act=act, slope=0.1, out=out, round_tf32=rnd)
            outs.append(out)
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1]), "run to run"
        assert torch.equal(outs[0], ref), (rnd, float((outs[0] - ref).abs().max()))


@pytest.mark.parametrize("shape", [(2, 256, 33, 65, 256), (1, 64, 9, 13, 136)])
def test_tma_epilogue_in_place_residual(shape):
    """out is the residual itself (the frozen bottleneck's conv3 adds in place)."""
    from structure_knowledge_distillation_b200 import ops
    N, Cin, H, W, Cout = shape
    x, w, sc, sh, g = _operands(N, Cin, H, W, Cout, 1, sum(shape))
    res0 = ops.to_nhwc(torch.randn(N, Cout, H, W, device="cuda", generator=g))
    raw = ops.conv2d_fwd(x, w, 1, 0, 1)
    ref = _reference(raw, sc, sh, res0, "relu", False)
    outs = []
    for _ in range(2):
        buf = res0.clone(memory_format=torch.channels_last)
        ops.conv2d_fwd(x, w, 1, 0, 1, scale=sc, shift=sh, residual=buf, act="relu", out=buf)
        outs.append(buf)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), "run to run"
    assert torch.equal(outs[0], ref), float((outs[0] - ref).abs().max())


@pytest.mark.parametrize("case", [(2, 64, 9, 13, 136, 1, 0), (1, 32, 10, 11, 200, 3, 2), (8, 256, 13, 21, 1024, 1, 0)])
def test_tma_epilogue_channel_slice_keeps_its_neighbours(case):
    """Output and residual are channel slices of wider buffers; every element outside the output slice, and every pixel past the
    last one, keeps its sentinel."""
    from structure_knowledge_distillation_b200 import ops
    N, Cin, H, W, Cout, k, pad = case
    x, w, sc, sh, g = _operands(N, Cin, H, W, Cout, k, sum(case))
    dil = 2 if k == 3 else 1
    oh, ow = ops.conv_out_hw(H, W, (k, k), 1, pad, dil)
    P, pitch, c_off = N * oh * ow, Cout + 44, 8
    res = ops.empty_nhwc(N, Cout + 12, oh, ow, "cuda")[:, 4:4 + Cout]
    res.copy_(torch.randn(N, Cout, oh, ow, device="cuda", generator=g))
    raw = ops.conv2d_fwd(x, w, 1, pad, dil)
    ref = _reference(raw, sc, sh, res, "relu", True)
    bufs = []
    for _ in range(2):
        buf, out = _sliced_out(N, Cout, oh, ow, pitch, c_off, 130)
        ops.conv2d_fwd(x, w, 1, pad, dil, scale=sc, shift=sh, residual=res, act="relu", out=out, round_tf32=True)
        bufs.append((buf, out))
    torch.cuda.synchronize()
    assert torch.equal(bufs[0][0], bufs[1][0]), "run to run"
    buf, out = bufs[0]
    assert torch.equal(out, ref), float((out - ref).abs().max())
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask.view(-1, pitch)[:P, c_off:c_off + Cout] = False
    assert bool((buf[mask] == SENTINEL).all()), int((buf[mask] != SENTINEL).sum())
