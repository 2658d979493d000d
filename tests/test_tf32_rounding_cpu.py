"""Host-side references for the layout, pooling and rounding kernel tests (tests/test_pool_layout_float64_gpu.py), each checked here
against hand-computed values so that the GPU tests compare against something already known to be right:

  * TF32 round-to-nearest-even on the float32 bit pattern (what `cvt.rn.tf32.f32` and a TFLOAT32 tensor map do),
    and the hi/lo split built on it;
  * the ceil-mode output size of the 3x3 / stride-2 / pad-1 max-pool, its forward with the first-maximum argmax, and the
    argmax-driven scatter of its backward;
  * im2col in the (kh, kw, ci) column order of skd_im2col_small.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F


# ---------------------------------------------------------------------------------------------- TF32 rounding
def rne_tf32_bits(u):
    """uint32 float32 bit patterns -> the TF32 value (low 13 mantissa bits zero) nearest to them, ties to even mantissa.
    Adding 0xFFF plus the lowest kept bit carries into bit 13 exactly when the dropped part is above half, or exactly half
    with an odd kept part; a carry out of the mantissa moves into the exponent (FLT_MAX rounds to Inf).  NaN and Inf pass."""
    u = np.asarray(u, dtype=np.uint32)
    special = (u & 0x7F800000) == 0x7F800000
    r = (u.astype(np.uint64) + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    return np.where(special, u, r.astype(np.uint32)).astype(np.uint32)


def round_tf32(x):
    x = np.ascontiguousarray(x, dtype=np.float32)
    return rne_tf32_bits(x.view(np.uint32)).view(np.float32)


def split_tf32(x):
    """-> (hi, lo) = (round_tf32(x), round_tf32(x - hi)), the difference taken in float32 as the kernel takes it."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = round_tf32(x)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = round_tf32(x - hi)
    return hi, lo


def tf32_special_values():
    """float32 bit patterns at the edges of TF32 rounding: ties of both parities and signs, just above / below a tie, subnormals,
    signed zeros, carries into the exponent, the largest finite value, Inf and NaN."""
    pats = [
        0x3F800000, 0x3F801000, 0x3F803000, 0x3F801001, 0x3F800FFF, 0x3F802FFF, 0x3F803001,    # 1.0 and ties around it
        0xBF801000, 0xBF803000, 0xBF801001, 0xBF800FFF,                                        # the same, negative
        0x3FFFF000, 0x3FFFFFFF, 0xBFFFF000, 0x3F7FF000,                                        # ties that carry into the exponent
        0x00000000, 0x80000000, 0x00000001, 0x00001000, 0x00003000, 0x00001001, 0x807FFFFF,    # zeros and subnormals
        0x007FF000, 0x007FFFFF, 0x00800000, 0x80001000,
        0x7F7FFFFF, 0xFF7FFFFF, 0x7F7FEFFF, 0x7F7FE000,                                        # largest finite values
        0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800001,                            # Inf, NaN (quiet and signalling)
    ]
    return np.array(pats, dtype=np.uint32)


@pytest.mark.parametrize("bits,want", [
    (0x3F800000, 0x3F800000),      # 1.0 is already TF32
    (0x3F801000, 0x3F800000),      # exact tie, even kept mantissa (...0) -> down
    (0x3F803000, 0x3F804000),      # exact tie, odd kept mantissa (...1) -> up to even
    (0x3F801001, 0x3F802000),      # just above the tie -> up
    (0x3F800FFF, 0x3F800000),      # just below the tie -> down
    (0xBF801000, 0xBF800000),      # negative tie, even -> magnitude down
    (0xBF803000, 0xBF804000),      # negative tie, odd -> magnitude up
    (0x3FFFF000, 0x40000000),      # 1.9995117 tie with odd mantissa -> carries into the exponent: 2.0
    (0x3FFFFFFF, 0x40000000),      # just below 2.0 -> 2.0
    (0x00000000, 0x00000000), (0x80000000, 0x80000000),      # +-0 keep their sign
    (0x00000001, 0x00000000),      # smallest subnormal -> +0
    (0x00001000, 0x00000000),      # subnormal tie, even -> 0
    (0x00003000, 0x00004000),      # subnormal tie, odd -> up
    (0x007FF000, 0x00800000),      # largest subnormal tie, odd -> carries into the smallest normal
    (0x7F7FFFFF, 0x7F800000),      # FLT_MAX -> +Inf
    (0xFF7FFFFF, 0xFF800000),      # -FLT_MAX -> -Inf
    (0x7F7FEFFF, 0x7F7FE000),      # below the tie under FLT_MAX stays finite
    (0x7F800000, 0x7F800000), (0xFF800000, 0xFF800000),      # Inf
])
def test_rne_tf32_hand_computed(bits, want):
    assert int(rne_tf32_bits(np.array([bits], dtype=np.uint32))[0]) == want


def test_rne_tf32_nan_stays_nan_and_low_bits_clear():
    v = tf32_special_values()
    r = rne_tf32_bits(v)
    f = v.view(np.float32)
    nan = np.isnan(f)
    assert np.all(np.isnan(r.view(np.float32)[nan]))
    assert np.all((r[~nan] & 0x1FFF) == 0)


def test_rne_tf32_is_nearest_on_random_bits():
    """Against float64 arithmetic: the result is one of the two TF32 neighbours and no farther than the other one."""
    rng = np.random.default_rng(0)
    u = rng.integers(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32)
    x = u.view(np.float32)
    keep = np.isfinite(x) & (np.abs(x) < 3.0e38)
    u, x = u[keep], x[keep].astype(np.float64)
    r = rne_tf32_bits(u).view(np.float32).astype(np.float64)
    down = (u & 0xFFFFE000).view(np.float32).astype(np.float64)
    up = ((u & 0xFFFFE000) + 0x2000).view(np.float32).astype(np.float64)
    assert np.all((r == down) | (r == up))
    err, other = np.abs(r - x), np.minimum(np.abs(down - x), np.abs(up - x))
    assert np.all(err <= other)


def test_split_tf32_bounds():
    """|x - hi - lo| <= 2^-21 |x| while lo is a normal number (|x| >= 2^-115): hi keeps 11 significant bits, lo the next 11 of
    the remaining 13.  Below that lo sits on the same absolute TF32 grid as hi (2^-136 below 2^-126: subnormals keep only their
    top 10 mantissa bits), so the remainder is bounded by half that step, 2^-137, not by one subnormal step (2^-149).
    FLT_MAX rounds up to Inf: hi = Inf, lo = -Inf, hi + lo = NaN (documented behaviour, not an accuracy case)."""
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(100000) * np.exp2(rng.integers(-140, 127, 100000))).astype(np.float32)
    x = x[np.abs(x) < 2.0 ** 127]
    hi, lo = split_tf32(x)
    res = np.abs(x.astype(np.float64) - hi.astype(np.float64) - lo.astype(np.float64))
    big = np.abs(x) >= np.float32(2.0 ** -115)
    assert big.sum() > 80000 and (~big).sum() > 1000
    assert np.all(res[big] <= 2.0 ** -21 * np.abs(x[big].astype(np.float64)))
    assert np.all(res[~big] <= 2.0 ** -137)
    sub = (np.arange(1, 2 ** 23, 9973, dtype=np.uint32)).view(np.float32)
    hi, lo = split_tf32(sub)
    assert np.all(np.abs(sub.astype(np.float64) - hi - lo) <= 2.0 ** -137)
    hi, lo = split_tf32(np.array([np.finfo(np.float32).max], dtype=np.float32))
    assert np.isposinf(hi[0]) and np.isneginf(lo[0])


# ---------------------------------------------------------------------------------------------- max-pool 3x3 / s2 / p1, ceil mode
def pool_out_ceil(n, k=3, s=2, p=1):
    """ATen pooling_output_shape with ceil_mode: the last window must start inside the input or its left padding."""
    o = (n + 2 * p - k + s - 1) // s + 1
    if (o - 1) * s >= n + p:
        o -= 1
    return o


def maxpool3x3s2_ref(x):
    """x: [N][H][W][C] float64 -> (y, argmax).  Taps visited in (ky, kx) order; a tap replaces the running maximum when it is
    strictly greater or NaN (F.max_pool2d's rule), so the argmax is the FIRST maximum and a NaN wins (the last NaN's index)."""
    n, h, w, c = x.shape
    oh, ow = pool_out_ceil(h), pool_out_ceil(w)
    pad = np.full((n, 2 * oh + 1, 2 * ow + 1, c), -np.inf)
    pad[:, 1:1 + h, 1:1 + w] = x[:, :2 * oh, :2 * ow]
    best = np.full((n, oh, ow, c), -np.inf)
    arg = np.zeros((n, oh, ow, c), dtype=np.uint8)
    for ky in range(3):
        for kx in range(3):
            v = pad[:, ky:ky + 2 * oh:2, kx:kx + 2 * ow:2]
            take = (v > best) | np.isnan(v)
            best = np.where(take, v, best)
            arg = np.where(take, np.uint8(ky * 3 + kx), arg)
    return best, arg


def maxpool3x3s2_bwd_ref(dy, arg, h, w):
    """dx[n][iy][ix][c] = sum of dy over the windows whose argmax is (iy, ix), in float64."""
    n, oh, ow, c = dy.shape
    pad = np.zeros((n, 2 * oh + 1, 2 * ow + 1, c))
    for ky in range(3):
        for kx in range(3):
            pad[:, ky:ky + 2 * oh:2, kx:kx + 2 * ow:2] += np.where(arg == ky * 3 + kx, dy, 0.0)
    return pad[:, 1:1 + h, 1:1 + w]


def test_pool_out_ceil_matches_torch():
    for n in list(range(1, 12)) + [256, 257, 512, 513]:
        assert pool_out_ceil(n) == F.max_pool2d(torch.zeros(1, 1, n, 1), (3, 1), (2, 1), (1, 0), ceil_mode=True).shape[2], n


def test_maxpool_ref_hand_computed():
    # 3x3 input, one channel: windows start at rows / cols -1 and 1 -> 2x2 output
    x = np.array([[1, 5, 5], [5, 2, 0], [3, 3, 3]], dtype=np.float64)[None, :, :, None]
    y, arg = maxpool3x3s2_ref(x)
    assert y[0, :, :, 0].tolist() == [[5, 5], [5, 3]]
    # window (0,0) covers rows -1..1, cols -1..1: the first 5 is at (row 0, col 1) = tap (ky=1, kx=2) = 5
    # window (0,1) covers rows -1..1, cols 1..3: first 5 at (0, 1) = tap (1, 0) = 3
    # window (1,0) covers rows 1..3, cols -1..1: first 5 at (1, 0) = tap (0, 1) = 1
    # window (1,1) covers rows 1..3, cols 1..3: max 3 first at (2, 1) = tap (1, 0) = 3
    assert arg[0, :, :, 0].tolist() == [[5, 3], [1, 3]]
    dy = np.array([[1.0, 2.0], [4.0, 8.0]])[None, :, :, None]
    dx = maxpool3x3s2_bwd_ref(dy, arg, 3, 3)[0, :, :, 0]
    assert dx.tolist() == [[0, 3, 0], [4, 0, 0], [0, 8, 0]]
    # NaN wins over every number, and a later NaN over an earlier one
    x = np.array([[1, np.nan], [np.nan, 7]], dtype=np.float64)[None, :, :, None]
    y, arg = maxpool3x3s2_ref(x)
    assert np.isnan(y[0, 0, 0, 0]) and arg[0, 0, 0, 0] == 7      # taps (1,1)=1, (1,2)=NaN, (2,1)=NaN, (2,2)=7 -> tap 7


def test_maxpool_ref_matches_torch():
    g = torch.Generator().manual_seed(0)
    for h, w in [(1, 1), (2, 5), (5, 4), (9, 13)]:
        x = torch.randint(-3, 4, (2, 6, h, w), generator=g).double()
        y, arg = maxpool3x3s2_ref(x.permute(0, 2, 3, 1).numpy())
        ty, tidx = F.max_pool2d(x, 3, 2, 1, ceil_mode=True, return_indices=True)
        assert np.array_equal(y, ty.permute(0, 2, 3, 1).numpy())
        # torch's flat index of the max, turned into the tap of each window
        oy = torch.arange(ty.shape[2])[:, None]; ox = torch.arange(ty.shape[3])[None, :]
        tap = ((tidx // w) - (2 * oy - 1)) * 3 + ((tidx % w) - (2 * ox - 1))
        assert np.array_equal(arg, tap.permute(0, 2, 3, 1).numpy().astype(np.uint8))


# ---------------------------------------------------------------------------------------------- im2col
def im2col_ref(x, kh, kw, stride, pad, dil, kp):
    """x: [N][H][W][Cin] -> [N][OH][OW][kp] with column (ky*kw + kx)*Cin + ci, zero outside the image and past KH*KW*Cin."""
    n, h, w, cin = x.shape
    oh = (h + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    ow = (w + 2 * pad - dil * (kw - 1) - 1) // stride + 1
    xp = np.zeros((n, h + 2 * pad + stride * oh, w + 2 * pad + stride * ow, cin), dtype=x.dtype)
    xp[:, pad:pad + h, pad:pad + w] = x
    col = np.zeros((n, oh, ow, kp), dtype=x.dtype)
    for ky in range(kh):
        for kx in range(kw):
            t = ky * kw + kx
            col[..., t * cin:(t + 1) * cin] = xp[:, ky * dil:ky * dil + stride * oh:stride, kx * dil:kx * dil + stride * ow:stride]
    return col


def test_im2col_ref_matches_unfold():
    g = torch.Generator().manual_seed(0)
    for (n, cin, h, w, k, s, p, d, kp) in [(2, 3, 7, 9, 3, 2, 1, 1, 28), (1, 5, 6, 5, 2, 1, 2, 2, 24)]:
        x = torch.randn(n, cin, h, w, generator=g, dtype=torch.float64)
        col = im2col_ref(x.permute(0, 2, 3, 1).numpy(), k, k, s, p, d, kp)
        u = F.unfold(x, k, dilation=d, padding=p, stride=s)                  # [N][ci*k*k + tap][L]
        oh, ow = col.shape[1:3]
        u = u.reshape(n, cin, k * k, oh, ow).permute(0, 3, 4, 2, 1).reshape(n, oh, ow, k * k * cin)
        assert np.array_equal(col[..., :k * k * cin], u.numpy())
        assert not col[..., k * k * cin:].any()
    # hand-computed: 1x2 image, 2 channels, 1x2 filter, no padding -> one output pixel [x00c0, x00c1, x01c0, x01c1, 0, 0]
    x = np.array([[[[1.0, 2.0], [3.0, 4.0]]]])
    assert im2col_ref(x, 1, 2, 1, 0, 1, 8)[0, 0, 0].tolist() == [1, 2, 3, 4, 0, 0, 0, 0]
