"""The NHWC ABN kernels (csrc/abn.cu: skd_abn_stats_nhwc, skd_abn_fold, skd_abn_apply_nhwc, skd_abn_bwd_reduce_nhwc,
skd_abn_bwd_dx_nhwc) against float64 at the student's own shapes.

At the benchmark configuration (batch 8, 512x1024 crops) the student's ABN layers see P = 1,048,576 rows (stem), 265,224 (after
the max-pool) and 67,080 (stride 8) with 64..512 channels.  These sizes take code paths the small shapes never reach: the 4-way
unrolled row loop of the statistics kernel, hundreds of row splits, and a grid-stride loop in the dx kernel that goes round many
times, with and without its one-channel-quad-per-thread shortcut.

Each stage is compared with a float64 restatement fed with what the previous stage produced (the apply pass with the kernel's
own scale / shift, the backward with its own mean / var), so a tolerance only has to cover the rounding of that stage.
Tolerances of sums are stated relative to the sum of the magnitudes of their terms.
"""
import numpy as np
import pytest
import torch

from test_tf32_rounding_cpu import round_tf32

pytestmark = pytest.mark.gpu

EPS, SLOPE, MOMENTUM = 1e-5, 0.01, 0.1
U = 2.0 ** -24                                 # unit roundoff of float32


@pytest.fixture(scope="module")
def ops():
    from structure_knowledge_distillation_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def L():
    from structure_knowledge_distillation_b200._cabi import lib
    return lib()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nhwc(t2d, n, h, w):
    """[P][C] rows -> (N, C, H, W) view of the same NHWC storage."""
    return t2d.view(n, h, w, -1).permute(0, 3, 1, 2)


def _geometry(L, P, C):
    """Launch geometry of the split-row reductions and of the dx kernel, as abn.cu computes it."""
    splits = L.skd_abn_num_splits(P, C)
    c4 = C // 4
    tr = 256 // min(c4, 256)
    rows_per = -(-P // splits)
    total4 = P * c4
    blocks = min(max(-(-total4 // 256), 1), 132 * 16)
    stride = blocks * 256
    return dict(splits=splits, tr=tr, rows_per=rows_per, unrolled=rows_per > 3 * tr, fixed_c=stride % c4 == 0,
                dx_loops=-(-total4 // stride), depth=-(-rows_per // tr) + tr + -(-splits // 32) + 8)


def _sum_tol(depth, abs_sum):
    """Recursive float32 summation: |error| <= (chain length) * u * sum|terms| (Higham, eq. 4.4).  `depth` bounds the longest
    chain of additions any term goes through: rows per thread, the block's row lanes, the splits per lane and the warp folds."""
    return depth * U * abs_sum


def _act64(pre, act):
    if act == "relu":
        return pre.clamp_min(0)
    if act == "leaky_relu":
        return torch.where(pre < 0, pre * SLOPE, pre)
    if act == "elu":
        return torch.where(pre < 0, torch.expm1(pre), pre)
    return pre


# ---------------------------------------------------------------------------------------------- statistics
STAT_SHAPES = [
    (1048576, 64),      # stem at 512x1024, batch 8
    (265224, 64),       # after the 3x3/s2 max-pool
    (67080, 128), (67080, 256), (67080, 512),      # stride 8
    (67080, 2048),      # two full 256-quad channel chunks
    (67080, 1028),      # a second channel chunk holding one quad
    (4096, 76), (3001, 260),                       # channel quads that are not a power of two (19, 65)
    (1, 64),            # one row: var = 0, running var keeps the biased value
    (21, 128),          # fewer than 32 rows: a single split
]


def _check_stats(st, rm, rv, rm0, rv0, x, w, b, P, label):
    xd = x.double()
    m64 = xd.mean(0)
    v64 = xd.var(0, unbiased=False)
    sd = v64.sqrt()
    mean, var, scale, shift = (t.double() for t in st)
    # requirement: mean within 1e-5 std, var within 1e-4 relative (or 1e-30 absolute for a constant channel)
    em = (mean - m64).abs() / sd.clamp_min(1e-30)
    ev = (var - v64).abs() / v64.clamp_min(1e-30)
    if P > 1:
        assert float(em.max()) <= 1e-5, (label, "mean", float(em.max()))
        assert float(ev.max()) <= 1e-4, (label, "var", float(ev.max()))
    else:
        assert torch.equal(st[0], x[0]) and torch.equal(st[1], torch.zeros_like(st[1])), label
    # running statistics: EMA of the float32 batch statistics; three float32 roundings of terms of size |rm0|, |mean|
    f = P / (P - 1) if P > 1 else 1.0
    ref_rm = rm0.double() * (1 - MOMENTUM) + MOMENTUM * m64
    ref_rv = rv0.double() * (1 - MOMENTUM) + MOMENTUM * f * v64
    tol_rm = MOMENTUM * 1e-5 * sd + 4 * U * (rm0.double().abs() + MOMENTUM * m64.abs())
    assert bool(((rm.double() - ref_rm).abs() <= tol_rm).all()), (label, "running_mean")
    tol_rv = MOMENTUM * f * 1e-4 * v64 + 5 * U * ref_rv.abs()
    assert bool(((rv.double() - ref_rv).abs() <= tol_rv).all()), (label, "running_var")
    # scale = (|w| + eps) / sqrt(var + eps): half of var's relative error plus three roundings
    gamma = w.double().abs() + EPS
    ref_sc = gamma / (v64 + EPS).sqrt()
    tol_sc = (0.5 * 1e-4 * v64 / (v64 + EPS) + 4 * U) * ref_sc
    assert bool(((scale - ref_sc).abs() <= tol_sc).all()), (label, "scale")
    # shift = b - mean * scale: the error of each factor, plus two roundings of terms of size |b|, |mean * scale|
    ref_sh = b.double() - m64 * ref_sc
    tol_sh = 1e-5 * sd * ref_sc + m64.abs() * tol_sc + 3 * U * (b.double().abs() + (m64 * ref_sc).abs())
    assert bool(((shift - ref_sh).abs() <= tol_sh).all()), (label, "shift")


@pytest.mark.parametrize("P,C", STAT_SHAPES)
def test_abn_stats_vs_float64(ops, P, C):
    g = _gen(P + C)
    x = torch.randn(P, C, device="cuda", generator=g) * 1.5 + 0.3
    w = torch.randn(C, device="cuda", generator=g)
    b = torch.randn(C, device="cuda", generator=g) * 0.2
    rm0 = torch.randn(C, device="cuda", generator=g) * 0.1
    rv0 = torch.rand(C, device="cuda", generator=g) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    st = ops.abn_stats(_nhwc(x, 1, 1, P), w, b, EPS, MOMENTUM, rm, rv)
    _check_stats(st, rm, rv, rm0, rv0, x, w, b, P, (P, C))


def test_abn_shapes_reach_every_reduction_path(L):
    """The shapes above and below drive each launch-geometry path: the unrolled row loop, more than 8 row splits, a single split,
    a partly filled second channel chunk, and dx grid-stride loops that repeat with and without the fixed-channel shortcut."""
    geo = {s: _geometry(L, *s) for s in STAT_SHAPES + [(P, C) for (_, P, C, *_rest) in BWD_CASES]}
    assert geo[(1048576, 64)]["unrolled"] and geo[(1048576, 64)]["splits"] > 8
    assert geo[(21, 128)]["splits"] == 1
    assert (1028 // 4) % 256 != 0
    assert any(g["fixed_c"] and g["dx_loops"] > 1 for g in geo.values())
    assert any(not g["fixed_c"] and g["dx_loops"] > 1 for g in geo.values())
    assert any(not g["fixed_c"] and g["dx_loops"] == 1 for g in geo.values())


def _data_class(name, P, C, g):
    std = 1.5
    if name == "normal":
        return torch.randn(P, C, device="cuda", generator=g) * std + 0.3
    if name == "post_relu":
        return torch.relu(torch.randn(P, C, device="cuda", generator=g))
    if name == "mean10_std0.1":
        return torch.randn(P, C, device="cuda", generator=g) * 0.1 + 10.0
    if name == "first_row_0_rest_8":
        x = torch.randn(P, C, device="cuda", generator=g) * 0.5 + 8.0
        x[0] = 0.0
        return x
    k = {"outlier_7sd": 7.0, "outlier_20sd": 20.0, "outlier_100sd": 100.0}[name]
    x = torch.randn(P, C, device="cuda", generator=g) * std + 0.3
    x[0] = 0.3 + k * std * torch.sign(torch.randn(C, device="cuda", generator=g))
    x[0, ::3] = x[1, ::3]                     # every third channel without the outlier: channel quads mix both cases
    return x


@pytest.mark.parametrize("name", ["normal", "post_relu", "mean10_std0.1", "first_row_0_rest_8", "outlier_7sd", "outlier_20sd",
                                  "outlier_100sd"])
@pytest.mark.parametrize("P,C", [(265224, 64), (67080, 512)])
def test_abn_stats_data_classes(ops, name, P, C):
    """The statistics are shifted by the channel's first row: a first row far from the mean must not cost precision."""
    g = _gen(7)
    x = _data_class(name, P, C, g)
    w = torch.randn(C, device="cuda", generator=g)
    b = torch.randn(C, device="cuda", generator=g)
    rm0, rv0 = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    rm, rv = rm0.clone(), rv0.clone()
    st = ops.abn_stats(_nhwc(x, 1, 1, P), w, b, EPS, MOMENTUM, rm, rv)
    _check_stats(st, rm, rv, rm0, rv0, x, w, b, P, name)


def test_abn_fold_vs_float64(ops):
    """Eval-mode / frozen-teacher folding: scale = (|w| + eps) / sqrt(var + eps), shift = b - mean * scale."""
    g = _gen(11)
    for C in (4, 64, 129 * 4, 2048):
        mean = torch.randn(C, device="cuda", generator=g) * 3
        var = torch.rand(C, device="cuda", generator=g) * 4
        var[0] = 0.0                                           # a dead channel: 1 / sqrt(eps)
        w = torch.randn(C, device="cuda", generator=g)
        b = torch.randn(C, device="cuda", generator=g)
        sc, sh = ops.abn_fold(mean, var, w, b, EPS)
        ref_sc = (w.double().abs() + EPS) / (var.double() + EPS).sqrt()
        # three roundings (|w| + eps, sqrt, the division) and the product: 4 u relative
        assert bool(((sc.double() - ref_sc).abs() <= 4 * U * ref_sc).all()), C
        ref_sh = b.double() - mean.double() * ref_sc
        assert bool(((sh.double() - ref_sh).abs() <= 6 * U * (b.double().abs() + (mean.double() * ref_sc).abs())).all()), C
        # without affine parameters: gamma = 1, beta = 0
        sc0, sh0 = ops.abn_fold(mean, var, None, None, EPS)
        ref0 = 1.0 / (var.double() + EPS).sqrt()
        assert bool(((sc0.double() - ref0).abs() <= 3 * U * ref0).all())
        assert bool(((sh0.double() + mean.double() * ref0).abs() <= 5 * U * (mean.double() * ref0).abs()).all())


# ---------------------------------------------------------------------------------------------- apply + backward
BWD_CASES = [
    # N, P = N*H*W, C, act, residual, chan_mul
    (8, 1048576, 64, "relu", False, False),         # stem: fixed-channel shortcut, the dx loop goes round 31 times
    (8, 265224, 64, "leaky_relu", True, False),
    (8, 67080, 128, "leaky_relu", False, True),     # Dropout2d mask, S = 8385 rows per image
    (8, 67080, 260, "elu", True, True),             # 65 quads: no shortcut, the dx loop repeats
    (8, 67080, 76, "none", False, True),            # 19 quads, likewise
    (8, 67080, 512, "relu", True, True),
    (8, 67080, 2048, "leaky_relu", False, False),   # two channel chunks
    (2, 4026, 1028, "elu", False, False),           # a partly filled second chunk
    (1, 1, 64, "leaky_relu", False, False),         # one row
    (1, 21, 128, "relu", True, True),               # one split
    (2, 234, 64, "elu", False, True),               # ELU with a mask that holds zeros (the stored output is masked)
]


def _inputs(N, P, C, res, drop, seed):
    g = _gen(seed)
    x = torch.randn(P, C, device="cuda", generator=g) * 1.5 + 0.3
    w = torch.randn(C, device="cuda", generator=g)
    b = torch.randn(C, device="cuda", generator=g) * 0.5
    r = torch.randn(P, C, device="cuda", generator=g) if res else None
    m = ((torch.rand(N, C, device="cuda", generator=g) > 0.3).float() / 0.7) if drop else None
    dout = torch.randn(P, C, device="cuda", generator=g)
    return x, w, b, r, m, dout


def _apply_ref(x, sc, sf, r, m, act, S):
    """float64 out and the magnitudes its float32 evaluation rounds: x*scale + shift (one FMA), + residual, act, * mask."""
    pre = x.double() * sc.double() + sf.double()
    mag = (x.double() * sc.double()).abs() + sf.double().abs()
    if r is not None:
        pre = pre + r.double()
        mag = mag + r.double().abs()
    o = _act64(pre, act)
    if m is not None:
        mm = m.double().repeat_interleave(S, 0)
        o, mag = o * mm, mag * mm.abs()
    return pre, o, mag


def _bwd_ref(x, out_k, dout, mean, var, w, m, act, S, training, P):
    """float64 ABN backward from the kernel's own mean / var and the activation branch of its own stored output."""
    mu, vv = mean.double(), var.double()
    invstd = 1.0 / (vv + EPS).sqrt()
    gamma = (w.double().abs() + EPS)
    y = (x.double() - mu) * invstd
    g = dout.double()
    o = out_k.double()
    if m is not None:
        mm = m.double().repeat_interleave(S, 0)
        g = g * mm
        o = torch.where(mm != 0, o / torch.where(mm != 0, mm, torch.ones_like(mm)), torch.zeros_like(o))
    if act == "relu":
        dz = torch.where(o > 0, g, torch.zeros_like(g))
    elif act == "leaky_relu":
        dz = torch.where(o < 0, g * SLOPE, g)
    elif act == "elu":
        dz = torch.where(o < 0, g * (o + 1), g)
    else:
        dz = g
    # what dz's own float32 evaluation may be off by: the mask product and the activation's factor round once each.  ELU's
    # factor o + 1 is formed from o near -1, so its error is u |g| however small exp(pre) = o + 1 is.
    dz_mag = g.abs() if act == "elu" else dz.abs()
    if training:
        s1, s2 = dz.sum(0), (dz * y).sum(0)
        a1, a2 = dz_mag.sum(0), (dz_mag * y.abs()).sum(0)
    else:
        s1 = s2 = a1 = a2 = torch.zeros_like(mu)
    edz, eydz = s1 / P, s2 / P
    k1 = gamma * invstd
    dx = (dz - edz - y * eydz) * k1
    mag = (dz_mag + edz.abs() + (y * eydz).abs()) * k1
    return dict(dz=dz, dz_mag=dz_mag, dx=dx, dx_mag=mag, y=y, k1=k1, s1=s1, s2=s2, a1=a1, a2=a2)


@pytest.mark.parametrize("N,P,C,act,res,drop", BWD_CASES)
def test_abn_apply_backward_vs_float64(ops, L, N, P, C, act, res, drop):
    S = P // N
    H, W = 1, S
    x, w, b, r, m, dout = _inputs(N, P, C, res, drop, seed=P + C)
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    xv = _nhwc(x, N, H, W)
    st = ops.abn_stats(xv, w, b, EPS, MOMENTUM, rm, rv)
    out = ops.abn_apply(xv, st[2], st[3], act, SLOPE, residual=_nhwc(r, N, H, W) if res else None, chan_mul=m)
    out2d = out.permute(0, 2, 3, 1).reshape(P, C)
    # forward: FMA, residual add, activation (expm1f: 2 ulp) and the mask each round once
    pre, o_ref, mag = _apply_ref(x, st[2], st[3], r, m, act, S)
    err = (out2d.double() - o_ref).abs()
    assert bool((err <= 4 * U * mag + 4 * U * o_ref.abs() + 1e-30).all()), ("out", float((err / mag.clamp_min(1e-30)).max()))
    # the activation branch the kernel took agrees with float64 wherever the pre-activation is not within rounding of 0
    if act != "none":
        mm = m.double().repeat_interleave(S, 0) if drop else torch.ones_like(pre)
        clear = (pre.abs() > 4 * U * mag / mm.abs().clamp_min(1e-30)) & (mm != 0)
        assert bool(((out2d > 0) == (pre > 0))[clear].all()) if act == "relu" else bool(((out2d < 0) == (pre < 0))[clear].all())
    # backward, batch statistics
    geo = _geometry(L, P, C)
    do4 = _nhwc(dout, N, H, W)
    dx, dres, dw, db = ops.abn_backward(xv, out, do4, st, w, EPS, act, SLOPE, m, res)
    ref = _bwd_ref(x, out2d, dout, st[0], st[1], w, m, act, S, True, P)
    # dbias = sum dz, dweight = sign(w) * sum y dz: float32 split sums (y itself rounds 3 times per term)
    # (each term carries dz's own 3 roundings)
    assert bool(((db.double() - ref["s1"]).abs() <= _sum_tol(geo["depth"] + 3, ref["a1"]) + 1e-30).all()), "dbias"
    sgn = torch.sign(w.double())
    assert bool(((dw.double() - sgn * ref["s2"]).abs() <= _sum_tol(geo["depth"] + 6, ref["a2"]) + 1e-30).all()), "dweight"
    # dx = k1 (dz - edz) - k2 (x - mean): a few roundings of each term plus the error of the two means it subtracts
    red = ref["k1"] * (_sum_tol(geo["depth"] + 3, ref["a1"]) + ref["y"].abs() * _sum_tol(geo["depth"] + 6, ref["a2"])) / P
    dx2d = dx.permute(0, 2, 3, 1).reshape(P, C)
    err = (dx2d.double() - ref["dx"]).abs()
    assert bool((err <= 8 * U * ref["dx_mag"] + red + 1e-30).all()), ("dx", float((err / (ref["dx_mag"] + red).clamp_min(1e-30)).max()))
    if res:
        # dres = dout * mask * act': the mask product and the activation's factor, 3 roundings at most
        assert bool(((dres.permute(0, 2, 3, 1).reshape(P, C).double() - ref["dz"]).abs() <= 3 * U * ref["dz_mag"]).all()), "dres"
    # TF32-rounded dx (it feeds a tensor-core convolution): bit for bit round_tf32 of the fp32 result
    dx_r, _, _, _ = ops.abn_backward(xv, out, do4, st, w, EPS, act, SLOPE, m, res, round_tf32=True)
    assert np.array_equal(dx_r.permute(0, 2, 3, 1).reshape(P, C).cpu().numpy(), round_tf32(dx2d.cpu().numpy())), "dx round_tf32"
    if not res and act != "elu":
        # the stored output not read: the sign recomputed from x*scale + shift, bit-identical results
        dx3, _, dw3, db3 = ops.abn_backward(xv, None, do4, st, w, EPS, act, SLOPE, m, False)
        assert torch.equal(dx3, dx) and torch.equal(dw3, dw) and torch.equal(db3, db)


@pytest.mark.parametrize("N,P,C,act", [(8, 67080, 256, "leaky_relu"), (8, 265224, 64, "relu"), (2, 4026, 260, "elu")])
def test_abn_eval_backward_vs_float64(ops, N, P, C, act):
    """training=False: stats are the running statistics, dx = dz * gamma / sqrt(running_var + eps), zero affine gradients."""
    S = P // N
    x, w, b, _, _, dout = _inputs(N, P, C, False, False, seed=P + 3)
    g = _gen(5)
    rmean = torch.randn(C, device="cuda", generator=g) * 0.3
    rvar = torch.rand(C, device="cuda", generator=g) * 2 + 0.5
    sc, sh = ops.abn_fold(rmean, rvar, w, b, EPS)
    st = torch.stack([rmean, rvar, sc, sh])
    xv = _nhwc(x, N, 1, S)
    out = ops.abn_apply(xv, sc, sh, act, SLOPE)
    out2d = out.permute(0, 2, 3, 1).reshape(P, C)
    dx, _, dw, db = ops.abn_backward(xv, out, _nhwc(dout, N, 1, S), st, w, EPS, act, SLOPE, None, False, training=False)
    ref = _bwd_ref(x, out2d, dout, rmean, rvar, w, None, act, S, False, P)
    err = (dx.permute(0, 2, 3, 1).reshape(P, C).double() - ref["dx"]).abs()
    assert bool((err <= 8 * U * ref["dx_mag"] + 1e-30).all())
    assert not dw.any() and not db.any()


@pytest.mark.parametrize("P,C,pitch,off", [(67080, 128, 384, 128), (265224, 64, 132, 68), (4026, 1028, 2048, 1020)])
def test_abn_apply_into_pitched_slice_and_tf32(ops, P, C, pitch, off):
    """out_pitch > C: the apply pass writes a channel slice of a wider buffer (the concat buffers of the PSP module) and leaves the
    other channels bit-identical; round_tf32 = 1 stores round_tf32 of the very same fp32 value."""
    x, w, b, r, m, _ = _inputs(8 if P % 8 == 0 else 2, P, C, True, True, seed=pitch)
    N = m.shape[0]
    S = P // N
    xv = _nhwc(x, N, 1, S)
    st = ops.abn_stats(xv, w, b, EPS, MOMENTUM, None, None)
    dense = ops.abn_apply(xv, st[2], st[3], "leaky_relu", SLOPE, residual=_nhwc(r, N, 1, S), chan_mul=m)
    sentinel = torch.tensor([0x7FC0ABCD], dtype=torch.int32).view(torch.float32).item()    # a NaN payload nothing computes
    buf = torch.full((P, pitch), sentinel, device="cuda")
    buf.view(torch.int32)[:, ::7] = -12345                                                     # and a second pattern
    before = buf.clone()
    view = _nhwc(buf, N, 1, S)[:, off:off + C]
    ops.abn_apply(xv, st[2], st[3], "leaky_relu", SLOPE, residual=_nhwc(r, N, 1, S), chan_mul=m, out=view)
    d2 = dense.permute(0, 2, 3, 1).reshape(P, C)
    assert torch.equal(buf[:, off:off + C].view(torch.int32), d2.contiguous().view(torch.int32))
    outside = torch.ones(pitch, dtype=torch.bool, device="cuda")
    outside[off:off + C] = False
    assert torch.equal(buf[:, outside].view(torch.int32), before[:, outside].view(torch.int32))
    rounded = ops.abn_apply(xv, st[2], st[3], "leaky_relu", SLOPE, residual=_nhwc(r, N, 1, S), chan_mul=m, round_tf32=True)
    assert np.array_equal(rounded.permute(0, 2, 3, 1).reshape(P, C).cpu().numpy(), round_tf32(d2.cpu().numpy()))
