"""Pooling, PSP-pyramid, layout and TF32-rounding kernels (csrc/pool.cu, csrc/conv_direct.cu, csrc/misc.cu) against float64 or
exact references, at the network's own map sizes and at the edges where index arithmetic goes wrong.

The references that are loops or bit manipulations (max-pool with its argmax, im2col, TF32 round-to-nearest-even) live in
tests/test_tf32_rounding_cpu.py and are checked there against hand-computed values.  Pooling and interpolation are compared with
float64 torch and its autograd adjoints; tolerances of sums are relative to the sum of the magnitudes of their terms.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_tf32_rounding_cpu import im2col_ref, maxpool3x3s2_bwd_ref, maxpool3x3s2_ref, rne_tf32_bits, split_tf32, tf32_special_values

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                                 # unit roundoff of float32


@pytest.fixture(scope="module")
def ops():
    from structure_knowledge_distillation_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def L():
    from structure_knowledge_distillation_b200._cabi import lib
    return lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nchw_view(buf):
    """[N][H][W][pitch] buffer -> (N, pitch, H, W) view."""
    return buf.permute(0, 3, 1, 2)


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy().view(np.uint32).ravel()


# ---------------------------------------------------------------------------------------------- max-pool 3x3 / s2 / p1, ceil mode
def _check_maxpool(ops, x, dy_seed):
    """x: (N, C, H, W) float32 on the GPU.  Forward bit-exact with F.max_pool2d, argmax equal to the first maximum in (ky, kx)
    order, backward exact against the float64 scatter through the same argmax (integer-valued dy: sums of <= 4 are exact)."""
    n, c, h, w = x.shape
    y, arg = ops.maxpool_fwd(ops.to_nhwc(x))
    ref = F.max_pool2d(x, 3, 2, 1, ceil_mode=True)
    assert y.shape == ref.shape
    assert torch.equal(y.isnan(), ref.isnan())
    assert torch.equal(torch.nan_to_num(y, nan=0.0), torch.nan_to_num(ref, nan=0.0))
    xr = x.permute(0, 2, 3, 1).double().cpu().numpy()
    _, arg_ref = maxpool3x3s2_ref(xr)
    assert np.array_equal(arg.cpu().numpy(), arg_ref)
    dy = torch.randint(-8, 9, ref.shape, device="cuda", generator=_gen(dy_seed)).float()
    dx = ops.maxpool_bwd(ops.to_nhwc(dy), arg, x.shape)
    dx_ref = maxpool3x3s2_bwd_ref(dy.permute(0, 2, 3, 1).double().cpu().numpy(), arg_ref, h, w)
    assert np.array_equal(dx.permute(0, 2, 3, 1).double().cpu().numpy(), dx_ref)


def test_maxpool_stem_shape_ties(ops):
    """The stem's 8x64x256x512 map, integer values in [-2, 2]: most windows hold several equal maxima."""
    x = torch.randint(-2, 3, (8, 64, 256, 512), device="cuda", generator=_gen(1)).float()
    _check_maxpool(ops, x, 2)


@pytest.mark.parametrize("H", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 5])
def test_maxpool_tiny_maps(ops, H, W):
    x = torch.randint(-1, 2, (2, 8, H, W), device="cuda", generator=_gen(10 * H + W)).float()
    _check_maxpool(ops, x, H + W)


def test_maxpool_nan_propagates_like_torch(ops):
    g = _gen(3)
    x = torch.randint(-2, 3, (2, 16, 13, 11), device="cuda", generator=g).float()
    x[torch.rand(x.shape, device="cuda", generator=g) < 0.05] = float("nan")
    x[0, 0, 0, 0] = float("nan")
    _check_maxpool(ops, x, 4)


# ---------------------------------------------------------------------------------------------- PSP pyramid
PSP_MAPS = [
    (8, 2048, 65, 129),     # the teacher's stride-8 map at 512x1024
    (8, 512, 97, 97),       # the student's, 769x769 crops
    (8, 512, 46, 61),       # 360x480 crops
    (1, 2048, 6, 6),        # one pixel per finest bin
    (1, 512, 1, 7), (1, 512, 7, 1),      # a single row / column
]
PSP_SIZES = [(1, 2, 3, 6), (6,), (1,)]


def _pool_tol_depth(h, w, s_count):
    """Longest float32 addition chain of one pooled value: a quarter row per lane, two shuffles, the segments of a bin, the rows."""
    return -(-w // 4) + 2 + 32 + h + 2


@pytest.mark.parametrize("sizes", PSP_SIZES)
@pytest.mark.parametrize("N,C,H,W", PSP_MAPS)
def test_psp_pool_fwd_bwd_vs_float64(ops, N, C, H, W, sizes):
    g = _gen(N + C + H + W)
    pitch, off = C + 512, 256                                  # x is a channel slice of a wider concat buffer
    buf = torch.randn(N, H, W, pitch, device="cuda", generator=g)
    x = _nchw_view(buf)[:, off:off + C]
    pooled = ops.psp_pool_fwd(x, list(sizes))
    xd = x.double()
    depth = _pool_tol_depth(H, W, len(sizes))
    at = 0
    for s in sizes:
        ref = F.adaptive_avg_pool2d(xd, (s, s))
        mag = F.adaptive_avg_pool2d(xd.abs(), (s, s))
        mine = pooled[:, at:at + s * s].reshape(N, s, s, C).permute(0, 3, 1, 2).double()
        # sum of <= area values then one division: depth * u of the mean magnitude, plus the division
        assert bool(((mine - ref).abs() <= (depth + 1) * U * mag).all()), (s, float(((mine - ref).abs() / mag).max()))
        at += s * s
    # backward: dx = sum over the bins holding the pixel of dpooled / area -- at most 4 bins per level, each term rounded twice
    dp = torch.randn(pooled.shape, device="cuda", generator=g)
    dx = ops.psp_pool_bwd(dp, list(sizes), (N, C, H, W))
    xr = xd.detach().clone().requires_grad_(True)
    tot, mag_tot, at = 0, 0, 0
    for s in sizes:
        p = F.adaptive_avg_pool2d(xr, (s, s))
        d = dp[:, at:at + s * s].reshape(N, s, s, C).permute(0, 3, 1, 2).double()
        tot = tot + (p * d).sum()
        mag_tot = mag_tot + (p * d.abs()).sum()
        at += s * s
    (gx,) = torch.autograd.grad(tot, xr, retain_graph=True)
    (gmag,) = torch.autograd.grad(mag_tot, xr)
    assert bool(((dx.double() - gx).abs() <= (4 * len(sizes) + 3) * U * gmag).all())


@pytest.mark.parametrize("sizes", PSP_SIZES)
@pytest.mark.parametrize("N,C,H,W", PSP_MAPS)
def test_psp_upsample_fwd_bwd_vs_float64(ops, N, C, H, W, sizes):
    g = _gen(3 * N + C + H + W)
    total = 4096
    chan_off = total - C - 4 * len(sizes)                     # a slice with untouched channels on both sides
    stage_all = torch.randn(N, sum(s * s for s in sizes), C, device="cuda", generator=g)
    at = 0
    for s in sizes:
        stage = stage_all[:, at:at + s * s].contiguous()
        at += s * s
        sd = stage.double().reshape(N, s, s, C).permute(0, 3, 1, 2)
        sentinel = torch.tensor([0x7FC0BEEF], dtype=torch.int32).view(torch.float32).item()
        out = torch.full((N, H, W, total), sentinel, device="cuda")
        out[..., ::5] = -3.25
        before = out.clone()
        ops.psp_upsample_fwd(stage, s, _nchw_view(out), chan_off)
        ref = F.interpolate(sd, size=(H, W), mode="bilinear", align_corners=True)
        mine = _nchw_view(out)[:, chan_off:chan_off + C].double()
        # source coordinate (s-1)/(H-1)*y rounds twice: weights off by <= 2 s u; then 3 roundings per corner product and sum
        vmax = sd.abs().amax((2, 3), keepdim=True)
        assert bool(((mine - ref).abs() <= (8 * s + 12) * U * vmax).all()), s
        outside = torch.ones(total, dtype=torch.bool, device="cuda")
        outside[chan_off:chan_off + C] = False
        assert torch.equal(out[..., outside].view(torch.int32), before[..., outside].view(torch.int32))
        # backward from a pitched dout: the adjoint of the same interpolation
        dout = torch.randn(N, H, W, total, device="cuda", generator=g)
        dstage = ops.psp_upsample_bwd(_nchw_view(dout), s, C, chan_off)
        sr = sd.detach().clone().requires_grad_(True)
        up = F.interpolate(sr, size=(H, W), mode="bilinear", align_corners=True)
        dsl = _nchw_view(dout)[:, chan_off:chan_off + C].double()
        (gs,) = torch.autograd.grad(up, sr, dsl)
        (gmag,) = torch.autograd.grad(F.interpolate(sr, size=(H, W), mode="bilinear", align_corners=True), sr, dsl.abs())
        mine_g = dstage.double().reshape(N, s, s, C).permute(0, 3, 1, 2)
        # float32 sums along a quarter row per lane and then down the rows, of terms w * dout; plus the weight error (2 s u per
        # weight) on every pixel of the image
        depth = -(-W // 4) + H + 8
        tol = depth * U * gmag + (2 * s + 4) * U * dsl.abs().sum((2, 3), keepdim=True)
        assert bool(((mine_g - gs).abs() <= tol).all()), s


# ---------------------------------------------------------------------------------------------- layout kernels
@pytest.mark.parametrize("rows,C,spitch,soff,dpitch,doff,src_shift", [
    (67080, 128, 384, 128, 256, 64, 0),        # float4 path
    (67080, 512, 4096, 3584, 1024, 0, 0),
    (4026, 19, 23, 3, 41, 5, 0),               # 19-class slices: scalar path
    (4026, 20, 20, 0, 64, 21, 0),              # destination offset not a multiple of 4
    (4026, 64, 64, 0, 128, 64, 1),             # everything a multiple of 4, but the source base is not 16-byte aligned
    (1, 4, 4, 0, 8, 4, 0),
])
def test_slice_copy_exact(ops, rows, C, spitch, soff, dpitch, doff, src_shift):
    g = _gen(rows + C)
    sflat = torch.randn(rows * spitch + src_shift, device="cuda", generator=g)
    src = _nchw_view(sflat[src_shift:].view(1, 1, rows, spitch))
    sentinel = torch.tensor([0x7FC01357], dtype=torch.int32).view(torch.float32).item()
    dst_buf = torch.full((1, 1, rows, dpitch), sentinel, device="cuda")
    before = dst_buf.clone()
    ops.slice_copy(src, soff, _nchw_view(dst_buf), doff, C)
    got = dst_buf[0, 0, :, doff:doff + C]
    want = sflat[src_shift:].view(rows, spitch)[:, soff:soff + C]
    assert torch.equal(got.contiguous().view(torch.int32), want.contiguous().view(torch.int32))
    outside = torch.ones(dpitch, dtype=torch.bool, device="cuda")
    outside[doff:doff + C] = False
    assert torch.equal(dst_buf[0, 0][:, outside].view(torch.int32), before[0, 0][:, outside].view(torch.int32))


def _ce_like_grad(P, C, ld, g):
    """softmax - one-hot rows: every row sums to 0, so column sums cancel between the label column and the others."""
    logits = torch.randn(P, C, device="cuda", generator=g) * 3
    lab = torch.randint(0, C, (P,), device="cuda", generator=g)
    d = torch.softmax(logits, 1)
    d[torch.arange(P, device="cuda"), lab] -= 1.0
    buf = torch.full((P, ld), float("nan"), device="cuda")        # the pitch padding must not be read
    buf[:, :C] = d / P
    return buf


@pytest.mark.parametrize("P,C,ld", [(4 * 2 ** 20, 19, 20), (2 ** 20, 19, 19), (67080, 512, 512), (67080, 100, 104), (31, 64, 64),
                                    (1, 19, 20)])
def test_colsum_vs_float64(L, P, C, ld):
    """db[c] (+)= sum over rows: 32 row lanes per column, each adding P/32 rows in float32, then 32 lane sums.  Bound: the
    probabilistic rounding-error bound 8 sqrt(chain) u sum|dy| (Higham & Mary 2019; 8 standard deviations) of the longest
    chain, P/32 + 32 additions."""
    g = _gen(P + C)
    dy = _ce_like_grad(P, C, ld, g)
    ref = dy[:, :C].double().sum(0)
    mag = dy[:, :C].double().abs().sum(0)
    tol = 8 * ((P / 32 + 32) ** 0.5) * U * mag
    db = torch.empty(C, device="cuda")
    L.skd_colsum(P, C, dy.data_ptr(), ld, db.data_ptr(), _st())
    assert bool(((db.double() - ref).abs() <= tol).all()), float(((db.double() - ref).abs() / mag).max())
    db0 = torch.randn(C, device="cuda", generator=g) * float(mag.mean())
    acc = db0.clone()
    L.skd_colsum_acc(P, C, dy.data_ptr(), ld, acc.data_ptr(), _st())
    # one more rounding, of the accumulated value
    assert bool(((acc.double() - db0.double() - ref).abs() <= tol + U * (db0.double() + ref).abs()).all())


@pytest.mark.parametrize("N,Cin,ldx,H,W,k,stride,pad,dil,kp", [
    (8, 3, 4, 512, 1024, 3, 2, 1, 1, 28),      # the stem: <3,3> instantiation, the image carried as 4 channels
    (2, 3, 3, 33, 17, 3, 1, 1, 1, 32),         # <3,3>, dense input, K padded from 27 to 32
    (2, 5, 8, 11, 13, 2, 1, 2, 2, 24),         # generic: 2x2, dilation 2
    (1, 3, 4, 9, 7, 5, 2, 2, 1, 76),           # generic: 5x5 over 3 channels
    (1, 4, 4, 1, 1, 3, 1, 1, 1, 36),           # one pixel: every tap but the centre is padding
])
def test_im2col_small_exact(ops, N, Cin, ldx, H, W, k, stride, pad, dil, kp):
    g = _gen(H + W + kp)
    buf = torch.randn(N, H, W, ldx, device="cuda", generator=g)
    x = _nchw_view(buf)[:, :Cin]
    col = ops.im2col_small(x, k, k, stride, pad, dil, kp)
    ref = im2col_ref(buf[..., :Cin].double().cpu().numpy(), k, k, stride, pad, dil, kp)
    assert np.array_equal(col.permute(0, 2, 3, 1).double().cpu().numpy(), ref)


@pytest.mark.parametrize("Cout,Cin,KH,KW", [(64, 128, 3, 3), (19, 512, 1, 1), (7, 5, 3, 2), (256, 64, 3, 3)])
def test_weight_flip_transpose_exact(L, Cout, Cin, KH, KW):
    """wt[ci][kh][kw][co] = w[co][KH-1-kh][KW-1-kw][ci]; with rounding, round_tf32 of exactly that value."""
    w = torch.randn(Cout, KH, KW, Cin, device="cuda", generator=_gen(Cout * Cin))
    want = w.flip(1, 2).permute(3, 1, 2, 0).contiguous()
    for rnd in (0, 1):
        wt = torch.empty(Cin, KH, KW, Cout, device="cuda")
        L.skd_weight_flip_transpose(Cout, Cin, KH, KW, w.data_ptr(), wt.data_ptr(), rnd, _st())
        exp = rne_tf32_bits(_bits(want)) if rnd else _bits(want)
        assert np.array_equal(_bits(wt), exp), rnd


# ---------------------------------------------------------------------------------------------- TF32 rounding
def _tf32_inputs():
    """Every special pattern, then random bit patterns (all exponents, NaN and Inf included), then random normals; a multiple
    of 4 long for the split kernel."""
    rng = np.random.default_rng(0)
    special = tf32_special_values()
    rand = rng.integers(0, 2 ** 32, 1 << 20, dtype=np.uint64).astype(np.uint32)
    ties = (rng.integers(0, 2 ** 19, 1 << 16, dtype=np.uint64).astype(np.uint32) << 13) | 0x1000      # exact ties, both parities
    u = np.concatenate([special, rand, ties])
    return u[: len(u) // 4 * 4]


def test_round_and_split_tf32_bit_exact(L):
    u = _tf32_inputs()
    x = torch.from_numpy(u.view(np.float32).copy()).cuda()
    n = x.numel()
    r = torch.empty_like(x)
    L.skd_round_tf32(n, x.data_ptr(), r.data_ptr(), _st())
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    L.skd_split_tf32(n, x.data_ptr(), hi.data_ptr(), lo.data_ptr(), _st())
    f = u.view(np.float32)
    nan = np.isnan(f)
    want = rne_tf32_bits(u)
    assert np.array_equal(_bits(r)[~nan], want[~nan])
    assert np.isnan(r.cpu().numpy()[nan]).all()
    assert np.array_equal(_bits(hi)[~nan], want[~nan])
    h_ref, l_ref = split_tf32(f)
    lo_bits, lr_bits = _bits(lo), l_ref.view(np.uint32)
    lnan = np.isnan(l_ref)
    assert np.array_equal(lo_bits[~lnan], lr_bits[~lnan])
    assert np.isnan(lo.cpu().numpy()[lnan]).all()
    # the split's documented edge: FLT_MAX rounds to hi = +Inf, lo = -Inf (hi + lo = NaN)
    i = int(np.nonzero(u == 0x7F7FFFFF)[0][0])
    assert np.isposinf(hi[i].item()) and np.isneginf(lo[i].item())
    # hi = NULL computes the same lo
    lo2 = torch.empty_like(x)
    L.skd_split_tf32(n, x.data_ptr(), None, lo2.data_ptr(), _st())
    assert torch.equal(lo2.view(torch.int32), lo.view(torch.int32))


def test_tfloat32_tensor_map_rounds_like_cvt_rn(ops, L):
    """The split-precision convolutions feed x_hi to the tensor cores as the TFLOAT32 tensor map's rounding of x and only store
    x_lo = round_tf32(x - round_tf32(x)).  That is exact only if the tensor map rounds to nearest even, as cvt.rn.tf32.f32 does.
    A 1x1 / stride-1 convolution takes the flat GEMM path, whose A operand (the activations) and B operand (the weights) are
    both loaded through tensor maps of the operand type; with an identity weight (exact in TF32) each output is the loaded x."""
    rng = np.random.default_rng(5)
    N, C, H, W = 2, 64, 32, 48
    P = N * H * W
    x = rng.standard_normal(P * C).astype(np.float32) * np.exp2(rng.integers(-60, 60, P * C)).astype(np.float32)
    u = x.view(np.uint32)
    u[: 1 << 14] = (u[: 1 << 14] & 0xFFFFE000) | 0x1000          # exact ties, both parities
    u[(1 << 14): (1 << 14) + 4096] |= 0x1FFF                      # the largest dropped part: carries
    xt = torch.from_numpy(x.copy()).cuda().view(N, H, W, C)
    w = torch.eye(C, device="cuda").view(C, 1, 1, C).contiguous()
    try:
        L.skd_set_tf32_tma_type(1)
        y = ops.conv2d_fwd(_nchw_view(xt), w, 1, 0, 1)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(y.permute(0, 2, 3, 1)), rne_tf32_bits(u))
        # FLOAT32 maps: the tensor core reads the low 13 bits as zero, so pre-rounded values pass through unchanged
        L.skd_set_tf32_tma_type(0)
        xr = torch.from_numpy(rne_tf32_bits(u).view(np.float32).copy()).cuda().view(N, H, W, C)
        y0 = ops.conv2d_fwd(_nchw_view(xr), w, 1, 0, 1)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(y0.permute(0, 2, 3, 1)), _bits(xr))
    finally:
        L.skd_set_tf32_tma_type(1)
