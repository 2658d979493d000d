"""Tensor-level wrappers over the C ABI (include/skd.h): pointer/stride plumbing only, no math.

Activations are torch tensors of logical shape (N, C, H, W) in channels-last memory (NHWC rows, optional row pitch
when the tensor is a channel slice of a wider buffer).  Everything runs on the caller's current CUDA stream.
"""
import math

import torch

from ._cabi import lib

ACT = {"none": 0, "leaky_relu": 1, "elu": 2, "relu": 3}

# bench.py sets this to a list to time every wgmma conv launch with CUDA events: (start, end, algorithmic FLOP)
CONV_EVENT_LOG = None


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _f32(*ts):
    for t in ts:
        if t is not None and t.dtype != torch.float32:
            raise TypeError("libskd_b200 kernels are fp32-storage only, got %s" % t.dtype)
        if t is not None and not t.is_cuda:
            raise RuntimeError("libskd_b200 has no CPU path: tensor is on %s" % t.device)


def empty_nhwc(n, c, h, w, device, pitch=None):
    """(N,C,H,W)-shaped view of a fresh NHWC buffer."""
    if pitch is None:
        return torch.empty((n, h, w, c), device=device, dtype=torch.float32).permute(0, 3, 1, 2)
    return torch.empty((n, h, w, pitch), device=device, dtype=torch.float32).permute(0, 3, 1, 2)[:, :c]


def pad4(c):
    return (c + 3) // 4 * 4


def pad_channels(t, cp):
    """(N,C,H,W) any layout -> dense NHWC tensor with cp >= C channels, zero-filled tail (TMA needs 16-byte pixel rows:
    the 3-channel image and the 19-class logits are carried as 4 / 20 channels)."""
    n, c, h, w = t.shape
    buf = torch.zeros((n, h, w, cp), device=t.device, dtype=torch.float32)
    buf[..., :c] = t.permute(0, 2, 3, 1)
    return buf.permute(0, 3, 1, 2)


def to_nhwc(t):
    """Any (N,C,H,W) tensor -> channels-last storage (no copy if it already is)."""
    return t.contiguous(memory_format=torch.channels_last) if t.dim() == 4 else t


def nhwc_meta(t):
    """-> (N, C, H, W, pitch) of an NHWC-stored (possibly channel-sliced) tensor; ValueError otherwise (functions.py:65-67)."""
    if t.dim() != 4:
        raise ValueError("Non-contiguous input")
    n, c, h, w = t.shape
    sn, sc, sh, sw = t.stride()
    # element (n,c,y,x) lives at n*sn + c + (y*w + x)*pitch; torch reports arbitrary strides for size-1 dims
    pitch = sw if w > 1 else (sh if h > 1 else (sn if n > 1 else c))
    ok = (c == 1 or sc == 1) and (w == 1 or sw == pitch) and (h == 1 or sh == w * pitch) and \
         (n == 1 or sn == h * w * pitch) and pitch >= c
    if not ok:
        raise ValueError("Non-contiguous input")
    return n, c, h, w, pitch


def pixel_strides(t):
    """(sn, sc, sp) over (image, channel, linear pixel) for NCHW-contiguous or NHWC(-pitched) tensors."""
    n, c, h, w = t.shape
    sn, sc, sh, sw = t.stride()
    if h > 1 and w > 1 and sh != w * sw:
        raise ValueError("Non-contiguous input")
    sp = sw if w > 1 else (sh if h > 1 else 1)
    return sn, sc, sp


# ------------------------------------------------------------------------------------------------ reference ABI (NCHW)
def bn_mean_var(x):
    _f32(x)
    if not x.is_contiguous():
        raise ValueError("Non-contiguous input")
    n, c = x.shape[0], x.shape[1]
    s = x.numel() // (n * c)
    mean = torch.empty(c, device=x.device); var = torch.empty(c, device=x.device)
    lib().skd_bn_mean_var_cuda(n, c, s, _p(x), _p(mean), _p(var), _st())
    return mean, var


# ------------------------------------------------------------------------------------------------ NHWC ABN
def abn_stats(x, weight, bias, eps, momentum, running_mean, running_var):
    n, c, h, w, pitch = nhwc_meta(x)
    if pitch != c:
        raise ValueError("Non-contiguous input")
    P = n * h * w
    L = lib()
    splits = L.skd_abn_num_splits(P, c)
    dev = x.device
    ws = torch.empty(splits * c * 6, device=dev)     # float (s1, s2) and double (s1, s2) partials per split and channel
    out = torch.empty(4, c, device=dev)              # mean, var, scale, shift
    L.skd_abn_stats_nhwc(P, c, _p(x), _p(weight), _p(bias), eps, momentum, _p(running_mean), _p(running_var),
                         _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]), _p(ws), splits, _st())
    return out


def abn_fold(mean, var, weight, bias, eps):
    c = mean.numel()
    out = torch.empty(2, c, device=mean.device)
    lib().skd_abn_fold(c, _p(mean), _p(var), _p(weight), _p(bias), eps, _p(out[0]), _p(out[1]), _st())
    return out[0], out[1]


def abn_apply(x, scale, shift, act, slope, residual=None, chan_mul=None, out=None, round_tf32=False):
    n, c, h, w, pitch = nhwc_meta(x)
    if pitch != c:
        raise ValueError("Non-contiguous input")
    if out is None:
        out = empty_nhwc(n, c, h, w, x.device)
    _, _, _, _, opitch = nhwc_meta(out)
    if residual is not None and nhwc_meta(residual)[4] != c:
        raise ValueError("Non-contiguous input")
    lib().skd_abn_apply_nhwc(n * h * w, c, h * w, _p(x), _p(out), opitch, _p(scale), _p(shift), ACT[act], slope,
                             _p(residual), _p(chan_mul), int(round_tf32), _st())
    return out


def abn_backward(x, out, dout, stats, weight, eps, act, slope, chan_mul, want_dres, round_tf32=False, training=True,
                 dweight_out=None, dbias_out=None, sync_fn=None):
    """-> dx, dres (or None), dweight, dbias.  dweight_out / dbias_out: write the affine gradients there (flat gradient views)."""
    n, c, h, w, pitch = nhwc_meta(x)
    if (out is not None and nhwc_meta(out)[4] != c) or nhwc_meta(dout)[4] != c or pitch != c:
        raise ValueError("Non-contiguous input")
    P = n * h * w
    L = lib()
    dev = x.device
    splits = L.skd_abn_num_splits(P, c)
    ws = torch.empty(splits * c * 2, device=dev)
    if training:
        red = torch.empty(4, c, device=dev)          # edz, eydz, dweight, dbias
        dwt = dweight_out if dweight_out is not None else red[2]
        dbt = dbias_out if dbias_out is not None else red[3]
        L.skd_abn_bwd_reduce_nhwc(P, c, h * w, _p(x), _p(out), _p(dout), _p(stats[0]), _p(stats[1]), _p(weight), eps, ACT[act],
                                  slope, _p(chan_mul), _p(red[0]), _p(red[1]), _p(dwt), _p(dbt), _p(ws), splits, _p(stats[2]), _p(stats[3]),
                                  _st())
        if sync_fn is not None:                      # synchronised statistics: edz / eydz are means over ALL ranks (functions.py:271-272)
            sync_fn(red[0:2])
    else:                                            # libs/functions.py:144-147: no batch-statistics terms, zero affine gradients
        red = torch.zeros(4, c, device=dev)
        dwt, dbt = red[2], red[3]
    dx = empty_nhwc(n, c, h, w, dev)
    dres = empty_nhwc(n, c, h, w, dev) if want_dres else None
    L.skd_abn_bwd_dx_nhwc(P, c, h * w, _p(x), _p(out), _p(dout), _p(dx), _p(dres), _p(stats[0]), _p(stats[1]), _p(weight),
                          _p(red[0]), _p(red[1]), eps, ACT[act], slope, _p(chan_mul), int(round_tf32), _p(stats[2]), _p(stats[3]), _st())
    return dx, dres, dwt, dbt


# ------------------------------------------------------------------------------------------------ convolutions
def conv_out_hw(h, w, k, stride, pad, dil):
    kh, kw = k
    return (h + 2 * pad - dil * (kh - 1) - 1) // stride + 1, (w + 2 * pad - dil * (kw - 1) - 1) // stride + 1


def weight_ohwi(weight):
    """(Cout,Cin,KH,KW) parameter -> its OHWI storage (channels-last weights need no copy)."""
    return weight.permute(0, 2, 3, 1).contiguous()      # no-op view when the parameter is channels_last


def conv2d_fwd(x, w_ohwi, stride, pad, dil, scale=None, shift=None, residual=None, act="none", slope=0.0,
               out=None, round_tf32=False, force_direct=False):
    """x: NHWC-stored (N,Cin,H,W) (pitch allowed); w_ohwi: contiguous [Cout][KH][KW][Cin]."""
    _f32(x, w_ohwi)
    n, cin, h, w, ldx = nhwc_meta(x)
    cout, kh, kw, cin2 = w_ohwi.shape
    assert cin2 == cin and w_ohwi.is_contiguous()
    oh, ow = conv_out_hw(h, w, (kh, kw), stride, pad, dil)
    if out is None:
        out = empty_nhwc(n, cout, oh, ow, x.device)
    on, oc, ooh, oow, ldy = nhwc_meta(out)
    assert (on, oc, ooh, oow) == (n, cout, oh, ow)
    L = lib()
    if force_direct or cin % 4 != 0 or ldx % 4 != 0:
        assert residual is None
        L.skd_conv2d_fwd_direct(n, h, w, cin, cout, kh, kw, stride, pad, dil, _p(x), ldx, _p(w_ohwi), _p(out), ldy, _p(scale),
                                _p(shift), ACT[act], slope, _st())
        return out
    ldr = nhwc_meta(residual)[4] if residual is not None else 0
    log = CONV_EVENT_LOG
    if log is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    L.skd_conv2d_fwd_sm100(n, h, w, cin, cout, kh, kw, stride, pad, dil, _p(x), ldx, _p(w_ohwi), _p(out), ldy, _p(scale),
                           _p(shift), _p(residual), ldr, ACT[act], slope, int(round_tf32), _st())
    if log is not None:
        ev1.record()
        log.append((ev0, ev1, 2.0 * n * oh * ow * cout * cin * kh * kw, ("fwd", n, cin, h, w, cout, kh, stride, dil)))
    return out


CHAIN_COUT1 = (64, 128, 256)


def conv1x1_chain_enabled():
    """skd_set_conv_chain: 0 (default) frozen bottlenecks chain conv3 into the next block's conv1, 1 never."""
    return lib().skd_conv_chain_mode() != 1


def conv1x1_chain(x3, w3_ohwi, scale3, shift3, residual, w1_ohwi, scale1, shift1, out3=None):
    """One launch for a frozen bottleneck's conv3 and the next block's conv1 (both 1x1, folded BN, ReLU):
    y3 = relu(conv(x3, w3) * scale3 + shift3 + residual), y1 = relu(conv(y3, w1) * scale1 + shift1) -> (y3, y1), each equal bit for
    bit to its conv2d_fwd.  out3 may be the residual."""
    _f32(x3, w3_ohwi, residual, w1_ohwi)
    n, cin3, h, w, ldx = nhwc_meta(x3)
    cout3, cout1 = w3_ohwi.shape[0], w1_ohwi.shape[0]
    assert w3_ohwi.shape == (cout3, 1, 1, cin3) and w1_ohwi.shape == (cout1, 1, 1, cout3)
    assert w3_ohwi.is_contiguous() and w1_ohwi.is_contiguous()
    if out3 is None:
        out3 = empty_nhwc(n, cout3, h, w, x3.device)
    assert nhwc_meta(out3)[:4] == (n, cout3, h, w) and nhwc_meta(residual)[:4] == (n, cout3, h, w)
    out1 = empty_nhwc(n, cout1, h, w, x3.device)
    log = CONV_EVENT_LOG
    if log is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    lib().skd_conv1x1_chain_sm100(n * h * w, cin3, cout3, cout1, _p(x3), ldx, _p(w3_ohwi), _p(scale3), _p(shift3), _p(residual),
                                  nhwc_meta(residual)[4], _p(out3), nhwc_meta(out3)[4], _p(w1_ohwi), _p(scale1), _p(shift1), _p(out1),
                                  cout1, _st())
    if log is not None:
        ev1.record()
        log.append((ev0, ev1, 2.0 * n * h * w * cout3 * (cin3 + cout1), ("fwd", n, cin3, h, w, cout3, "chain1x1->%d" % cout1)))
    return out3, out1


def lo_tf32(t):
    """dense tensor -> lo = rna_tf32(t - rna_tf32(t)), same layout (the hi part is what a TFLOAT32 tensor map makes of t itself)."""
    lo = torch.empty_strided(t.shape, t.stride(), device=t.device, dtype=torch.float32)
    lib().skd_split_tf32(t.numel(), _p(t), None, _p(lo), _st())
    return lo


def conv2d_fwd_3xtf32(x, w_ohwi, stride, pad, dil, shift=None):
    """fp32-grade forward convolution: split-precision operands, three tensor-core passes in one launch."""
    n, cin, h, w, ldx = nhwc_meta(x)
    if ldx != cin:
        raise ValueError("Non-contiguous input")
    cout, kh, kw, _ = w_ohwi.shape
    oh, ow = conv_out_hw(h, w, (kh, kw), stride, pad, dil)
    out = empty_nhwc(n, cout, oh, ow, x.device)
    log = CONV_EVENT_LOG
    if log is not None:
        ev0, ev1, ev2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        ev0.record()
    xh, xl = x, lo_tf32(x)
    wh, wl = w_ohwi, lo_tf32(w_ohwi)
    if log is not None:
        ev1.record()
    lib().skd_conv2d_fwd_sm100_3xtf32(n, h, w, cin, cout, kh, kw, stride, pad, dil, _p(xh), _p(xl), ldx, _p(wh), _p(wl), _p(out), cout,
                                      None, _p(shift), 0, 0.0, _st())
    if log is not None:
        ev2.record()
        log.append((ev0, ev1, 0.0, ("split3x", n, cin, h, w, cout, kh, stride, dil)))
        # ALGORITHMIC flop (1x): the two extra split-precision passes are an implementation cost, not work the reference does
        log.append((ev1, ev2, 2.0 * n * oh * ow * cout * cin * kh * kw, ("fwd3x", n, cin, h, w, cout, kh, stride, dil)))
    return out


def conv2d_dgrad(dy, w_ohwi, x_shape, stride, pad, dil, round_tf32=False, force_direct=False, residual=None):
    """dx for y = conv(x, w).  stride 1: forward wgmma kernel on dy with the flipped/transposed weights.  `residual` (stride-1
    wgmma path only): dx + residual, added by the kernel's epilogue -- the fixed-order sum of several data gradients into one
    tensor (ESPNet-C's branches)."""
    n, cin, h, w = x_shape
    cout, kh, kw, _ = w_ohwi.shape
    L = lib()
    dn, dc, doh, dow, ldy = nhwc_meta(dy)
    dx = empty_nhwc(n, cin, h, w, dy.device)
    wgmma = stride == 1 and not force_direct and cout % 4 == 0 and ldy % 4 == 0
    if residual is not None and not (wgmma and cin % 4 == 0):
        raise ValueError("conv2d_dgrad: a residual needs the stride-1 wgmma path (channel counts padded to multiples of 4)")
    ldr = nhwc_meta(residual)[4] if residual is not None else 0
    if wgmma:
        wt = torch.empty((cin, kh, kw, cout), device=dy.device, dtype=torch.float32)
        L.skd_weight_flip_transpose(cout, cin, kh, kw, _p(w_ohwi), _p(wt), 0, _st())
        log = CONV_EVENT_LOG
        if log is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        L.skd_conv2d_fwd_sm100(n, doh, dow, cout, cin, kh, kw, 1, dil * (kh - 1) - pad, dil, _p(dy), ldy, _p(wt), _p(dx), cin,
                               None, None, _p(residual), ldr, 0, 0.0, int(round_tf32), _st())
        if log is not None:
            ev1.record()
            log.append((ev0, ev1, 2.0 * n * h * w * cin * cout * kh * kw, ("dgrad", n, cout, doh, dow, cin, kh, 1, dil)))
    elif stride == 2 and dil == 1 and not force_direct and cout % 4 == 0 and ldy % 4 == 0 and cin % 4 == 0:
        # dgrad of a stride-2 convolution = one stride-1 convolution of dy per input-pixel parity class (py, px): the taps
        # with (py + pad - kh) even, taken in descending kh order, written to the every-other-pixel sub-grid of dx
        dx.zero_()                                           # classes without a tap (1x1 stride-2: odd rows/cols) stay zero
        for py in range(2):
            khs = [k for k in range(kh) if (py + pad - k) % 2 == 0]
            if not khs or py >= h:
                continue
            for px in range(2):
                kws = [k for k in range(kw) if (px + pad - k) % 2 == 0]
                if not kws or px >= w:
                    continue
                ty, tx = [(py + pad - k) // 2 for k in khs], [(px + pad - k) // 2 for k in kws]
                khs_d, kws_d = khs[::-1], kws[::-1]          # ascending offset t <-> descending tap index
                pad_y, pad_x = -min(ty), -min(tx)
                assert pad_y == pad_x, "asymmetric sub-kernel padding is not supported"
                wsub = torch.stack([w_ohwi[:, a] for a in khs_d], 1)               # device-side gathers only (graph capturable)
                wsub = torch.stack([wsub[:, :, b] for b in kws_d], 2)              # [Cout][KH'][KW'][Cin]
                wt = wsub.permute(3, 1, 2, 0).contiguous()   # [Cin][KH'][KW'][Cout]
                hc, wc = (h - py + 1) // 2, (w - px + 1) // 2
                view = dx[:, :, py::2, px::2]
                # output extent = size of the parity class; taps that fall past dy's edge read hardware zero fill
                L.skd_conv2d_fwd_sm100_strided(n, doh, dow, cout, cin, len(khs), len(kws), 1, pad_y, 1, _p(dy), ldy, _p(wt),
                                               view.data_ptr(), view.stride(3), view.stride(2), view.stride(0), hc, wc,
                                               int(round_tf32), _st())
    else:
        L.skd_conv2d_dgrad_direct(n, h, w, cin, cout, kh, kw, stride, pad, dil, _p(dy), ldy, _p(w_ohwi), _p(dx), cin, _st())
    return dx


def conv2d_wgrad(x, dy, kshape, stride, pad, dil, force_direct=False, out=None):
    """dw in OHWI layout [Cout][KH][KW][Cin] (written into `out` when given: a dense OHWI buffer of that size)."""
    n, cin, h, w, ldx = nhwc_meta(x)
    dn, cout, doh, dow, ldy = nhwc_meta(dy)
    kh, kw = kshape
    L = lib()
    dw = out if out is not None else torch.empty((cout, kh, kw, cin), device=x.device, dtype=torch.float32)
    if force_direct or cin % 4 or cout % 4 or ldx % 4 or ldy % 4:
        L.skd_conv2d_wgrad_direct(n, h, w, cin, cout, kh, kw, stride, pad, dil, _p(x), ldx, _p(dy), ldy, _p(dw), _st())
    else:
        nws = L.skd_conv2d_wgrad_sm100_workspace_floats(n, h, w, cin, cout, kh, kw, stride, pad, dil)
        ws = torch.empty(max(nws, 4), device=x.device, dtype=torch.float32)
        log = CONV_EVENT_LOG
        if log is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        L.skd_conv2d_wgrad_sm100(n, h, w, cin, cout, kh, kw, stride, pad, dil, _p(x), ldx, _p(dy), ldy, _p(dw), _p(ws), _st())
        if log is not None:
            ev1.record()
            log.append((ev0, ev1, 2.0 * n * doh * dow * cout * cin * kh * kw, ("wgrad", n, cin, h, w, cout, kh, stride, dil)))
    return dw


def conv_transpose2x2_fwd(x, w_rows):
    """nn.ConvTranspose2d(k=2, stride=2, no bias) forward, fp32-grade (3xTF32).  x: dense NHWC (N, Cin, h, w), Cin a multiple of 4;
    w_rows: contiguous [2][2 * Coutp][1][1][Cin] -- for output-row parity a, the 1x1 weights of the two output columns 2j, 2j + 1
    stacked (Coutp each).  Output pixels (2i + a, 2j) and (2i + a, 2j + 1) are 2 * Coutp consecutive floats, so each parity is one
    1x1 GEMM to 2 * Coutp channels written onto the every-other-row sub-grid.  -> dense NHWC (N, Coutp, 2h, 2w)."""
    n, cin, h, w, ldx = nhwc_meta(x)
    if ldx != cin or cin % 4:
        raise ValueError("Non-contiguous input")
    cout2 = w_rows.shape[1]
    coutp = cout2 // 2
    y = empty_nhwc(n, coutp, 2 * h, 2 * w, x.device)
    xl, wl = lo_tf32(x), lo_tf32(w_rows)
    base = y.data_ptr()
    log = CONV_EVENT_LOG
    if log is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    for a in range(2):
        lib().skd_conv2d_fwd_sm100_strided_3xtf32(n, h, w, cin, cout2, 1, 1, 1, 0, 1, _p(x), _p(xl), ldx, _p(w_rows[a]), _p(wl[a]),
                                                  base + 4 * a * 2 * w * coutp, cout2, 4 * w * coutp, 4 * h * w * coutp, _st())
    if log is not None:
        ev1.record()
        log.append((ev0, ev1, 2.0 * n * h * w * cin * 4 * coutp, ("convT_fwd", n, cin, h, w, coutp, 2, 2, 1)))
    return y


def im2col_small(x, kh, kw, stride, pad, dil, kp):
    """(N,Cin,H,W) NHWC-stored -> (N, kp, OH, OW) NHWC-stored im2col matrix (k = tap*Cin + ci, zero padded)."""
    n, cin, h, w, ldx = nhwc_meta(x)
    oh, ow = conv_out_hw(h, w, (kh, kw), stride, pad, dil)
    col = empty_nhwc(n, kp, oh, ow, x.device)
    lib().skd_im2col_small(n, h, w, cin, kh, kw, stride, pad, dil, _p(x), ldx, _p(col), kp, _st())
    return col


def colsum(dy, out=None):
    n, c, h, w, ld = nhwc_meta(dy)
    db = out if out is not None else torch.empty(c, device=dy.device, dtype=torch.float32)
    lib().skd_colsum(n * h * w, c, _p(dy), ld, _p(db), _st())
    return db


# ------------------------------------------------------------------------------------------------ pooling
def maxpool_fwd(x):
    n, c, h, w, pitch = nhwc_meta(x)
    if pitch != c:
        raise ValueError("Non-contiguous input")
    L = lib()
    oh, ow = L.skd_pool_out_size_ceil(h, 3, 2, 1), L.skd_pool_out_size_ceil(w, 3, 2, 1)
    y = empty_nhwc(n, c, oh, ow, x.device)
    arg = torch.empty((n, oh, ow, c), device=x.device, dtype=torch.uint8)
    L.skd_maxpool3x3s2_fwd(n, h, w, c, _p(x), _p(y), _p(arg), _st())
    return y, arg


def maxpool_bwd(dy, arg, x_shape):
    n, c, h, w = x_shape
    if nhwc_meta(dy)[4] != c:
        raise ValueError("Non-contiguous input")
    dx = empty_nhwc(n, c, h, w, dy.device)
    lib().skd_maxpool3x3s2_bwd(n, h, w, c, _p(dy), _p(arg), _p(dx), _st())
    return dx


def _sizes_arr(sizes):
    import ctypes
    return (ctypes.c_int * len(sizes))(*sizes)


def psp_pool_fwd(x, sizes):
    n, c, h, w, pitch = nhwc_meta(x)
    nb = sum(s * s for s in sizes)
    pooled = torch.empty((n, nb, c), device=x.device, dtype=torch.float32)
    arr = _sizes_arr(sizes)
    import ctypes
    ap = ctypes.cast(arr, ctypes.c_void_p)
    ws = torch.empty(lib().skd_psp_pool_workspace_floats(n, h, c, len(sizes), ap), device=x.device, dtype=torch.float32)
    lib().skd_psp_pool_fwd(n, h, w, c, _p(x), pitch, len(sizes), ap, _p(pooled), _p(ws), _st())
    return pooled


def psp_pool_bwd(dpooled, sizes, x_shape):
    n, c, h, w = x_shape
    dx = empty_nhwc(n, c, h, w, dpooled.device)
    arr = _sizes_arr(sizes)
    import ctypes
    lib().skd_psp_pool_bwd(n, h, w, c, _p(dpooled), len(sizes), ctypes.cast(arr, ctypes.c_void_p), _p(dx), _st())
    return dx


def psp_upsample_fwd(stage, s, out, chan_off):
    """stage: (N, s*s, C) contiguous -> out[:, chan_off:chan_off+C] (NHWC buffer, in place)."""
    n, nb, c = stage.shape
    on, oc, h, w, pitch = nhwc_meta(out)
    lib().skd_psp_upsample_fwd(n, h, w, c, s, _p(stage), nb, 0, _p(out), pitch, chan_off, _st())


def psp_upsample_bwd(dout, s, c, chan_off):
    n, ctot, h, w, pitch = nhwc_meta(dout)
    dstage = torch.empty((n, s * s, c), device=dout.device, dtype=torch.float32)
    ws = torch.empty(lib().skd_psp_upsample_bwd_workspace_floats(n, h, c, s), device=dout.device, dtype=torch.float32)
    lib().skd_psp_upsample_bwd(n, h, w, c, s, _p(dout), pitch, chan_off, _p(dstage), s * s, 0, _p(ws), _st())
    return dstage


def slice_copy(src, src_off, dst, dst_off, c):
    n, _, h, w, sp = nhwc_meta(src)
    dp = nhwc_meta(dst)[4]
    lib().skd_slice_copy(n * h * w, c, _p(src), sp, src_off, _p(dst), dp, dst_off, _st())


# ------------------------------------------------------------------------------------------------ losses
def _ws(device, n=None):
    n = n or 2 * lib().skd_loss_max_partials()
    return torch.empty(n, device=device, dtype=torch.float64)


def pixelwise_fwd(S, T):
    _f32(S, T)
    n, c, h, w = S.shape
    loss = torch.empty((), device=S.device, dtype=torch.float32)
    # reference quirk: N,C,W,H = shape and /W/H  (utils/criterion.py:222,225) == / (shape[2]*shape[3])
    lib().skd_pixelwise_fwd(n, c, h * w, _p(S), *pixel_strides(S), _p(T), *pixel_strides(T), 1.0 / (h * w), _p(loss),
                            _p(_ws(S.device)), _st())
    return loss


def pixelwise_bwd(S, T, grad_out):
    n, c, h, w = S.shape
    dS = torch.empty_strided(S.shape, S.stride(), device=S.device, dtype=torch.float32)   # same layout as S
    lib().skd_pixelwise_bwd(n, c, h * w, _p(S), *pixel_strides(S), _p(T), *pixel_strides(T), _p(dS), *pixel_strides(dS),
                            _p(grad_out), 1.0 / (h * w), _st())
    return dS


def at_fwd(S, T):
    """Attention transfer (csrc/feature_kd.cu) of NHWC-stored (pitch allowed) student / teacher maps on one grid -> (loss, qhat
    (2, N*H*W): the normalised maps of S and T, norms (2, N): the per-sample norms of the unnormalised maps)."""
    _f32(S, T)
    n, cs, h, w, lds = nhwc_meta(S)
    nt, ct, ht, wt, ldt = nhwc_meta(T)
    if (nt, ht, wt) != (n, h, w):
        raise ValueError("attention transfer: student %s and teacher %s maps differ in batch or grid" % (tuple(S.shape), tuple(T.shape)))
    qhat = torch.empty((2, n * h * w), device=S.device, dtype=torch.float32)
    norms = torch.empty((2, n), device=S.device, dtype=torch.float32)
    loss = torch.empty((), device=S.device, dtype=torch.float32)
    lib().skd_at_fwd(n, h * w, cs, _p(S), lds, ct, _p(T), ldt, _p(qhat), _p(norms), _p(loss), _st())
    return loss, qhat, norms


def at_bwd(S, qhat, norms, grad_out):
    """d loss / d S of at_fwd, in S's layout."""
    n, c, h, w, lds = nhwc_meta(S)
    dS = torch.empty_strided(S.shape, S.stride(), device=S.device, dtype=torch.float32)
    g = torch.empty(n * h * w, device=S.device, dtype=torch.float32)
    lib().skd_at_bwd(n, h * w, c, _p(S), lds, _p(qhat), _p(norms), _p(grad_out), _p(g), _p(dS), lds, _st())
    return dS


def mse_fwd(R, T):
    """F.mse_loss(R, T) of NHWC-stored (pitch allowed) maps of one shape (csrc/feature_kd.cu)."""
    _f32(R, T)
    if tuple(R.shape) != tuple(T.shape):
        raise ValueError("mse: shapes %s and %s differ" % (tuple(R.shape), tuple(T.shape)))
    n, c, h, w, ldr = nhwc_meta(R)
    loss = torch.empty((), device=R.device, dtype=torch.float32)
    lib().skd_mse_fwd(n * h * w, c, _p(R), ldr, _p(T), nhwc_meta(T)[4], _p(loss), _p(_ws(R.device)), _st())
    return loss


def mse_bwd(R, T, grad_out):
    """d mse_fwd(R, T) / d R, dense NHWC."""
    n, c, h, w, ldr = nhwc_meta(R)
    dR = empty_nhwc(n, c, h, w, R.device)
    lib().skd_mse_bwd(n * h * w, c, _p(R), ldr, _p(T), nhwc_meta(T)[4], _p(grad_out), _p(dR), c, _st())
    return dR


def _cwd_check(S, T, tau):
    if S.dim() != 4 or tuple(T.shape) != tuple(S.shape):
        raise ValueError("channel-wise distillation: student %s and teacher %s maps differ in batch, channels or grid"
                         % (tuple(S.shape), tuple(T.shape)))
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError("channel-wise distillation: the temperature must be finite and > 0 (got %r)" % (tau,))


def cwd_fwd(S, T, tau):
    """Channel-wise distillation (csrc/cwd.cu) of student / teacher maps of one (N, C, H, W) shape, NCHW or NHWC (pitch allowed) ->
    (loss, lse (2, N, C) float64: the log-sum-exp of x / tau over H*W per (map, image, channel), what the backward reads)."""
    _f32(S, T)
    _cwd_check(S, T, tau)
    n, c, h, w = S.shape
    loss = torch.empty((), device=S.device, dtype=torch.float32)
    lse = torch.empty((2, n, c), device=S.device, dtype=torch.float64)
    ws = _ws(S.device, lib().skd_cwd_workspace(n, c, h * w))
    lib().skd_cwd_fwd(n, c, h * w, _p(S), *pixel_strides(S), _p(T), *pixel_strides(T), float(tau), _p(loss), _p(lse), _p(ws), _st())
    return loss, lse


def cwd_bwd(S, T, lse, tau, grad_out):
    """d loss / d S of cwd_fwd, in S's layout."""
    _cwd_check(S, T, tau)
    n, c, h, w = S.shape
    dS = torch.empty_strided(S.shape, S.stride(), device=S.device, dtype=torch.float32)
    lib().skd_cwd_bwd(n, c, h * w, _p(S), *pixel_strides(S), _p(T), *pixel_strides(T), float(tau), _p(lse), _p(grad_out), _p(dS),
                      *pixel_strides(dS), _st())
    return dS


def _labels_check(labels, n):
    if labels.dtype != torch.int64 or labels.dim() != 3 or not labels.is_contiguous():
        raise ValueError("labels must be a contiguous (N, H, W) int64 tensor (got %s %s%s)"
                         % (labels.dtype, tuple(labels.shape), "" if labels.is_contiguous() else ", not contiguous"))
    if n is not None and labels.shape[0] != n:
        raise ValueError("labels hold %d images for a batch of %d" % (labels.shape[0], n))


def labels_nearest(labels, h, w):
    """(N, H, W) int64 labels on the device -> (N, h, w) int32, each the label F.interpolate(labels[:, None].float(), (h, w),
    mode="nearest") picks (torch's legacy rule src = min(floor(dst * (float(in) / out)), in - 1) in fp32); labels outside the int32
    range become -1."""
    _labels_check(labels, None)
    if not labels.is_cuda:
        raise RuntimeError("libskd_b200 has no CPU path: tensor is on %s" % labels.device)
    if h < 1 or w < 1:
        raise ValueError("labels_nearest: empty grid %dx%d" % (h, w))
    n, H, W = labels.shape
    out = torch.empty((n, h, w), device=labels.device, dtype=torch.int32)
    lib().skd_labels_nearest(n, H, W, _p(labels), h, w, _p(out), _st())
    return out


def _ifv_check(S, T, labels, classes_num):
    if S.dim() != 4 or T.dim() != 4 or S.shape[0] != T.shape[0] or tuple(S.shape[2:]) != tuple(T.shape[2:]):
        raise ValueError("intra-class variation: student %s and teacher %s maps differ in batch or grid"
                         % (tuple(S.shape), tuple(T.shape)))
    _labels_check(labels, S.shape[0])
    if not 1 <= classes_num <= 255:
        raise ValueError("intra-class variation: the class count must be in [1, 255] (got %r)" % (classes_num,))


def _row_strides(t):
    """(sn, sp) of an NHWC-stored (pitch allowed) map."""
    n, c, h, w, pitch = nhwc_meta(t)
    return h * w * pitch, pitch


def ifv_fwd(S, T, labels, classes_num):
    """Intra-class feature variation distillation (csrc/ifv.cu) of NHWC-stored (pitch allowed) student / teacher maps on one grid, with
    the step's (N, H, W) int64 labels -> (loss, saved): `saved` = (lab (N, h, w) int32 from labels_nearest, P_S (N, K, C_S) fp32, stats
    (3, N, K) float64: counts, |P_S|^2, |P_T|^2, pix (3, N, h*w) fp32: cos_S, cos_S - cos_T, |f_S|), what ifv_bwd reads."""
    _f32(S, T)
    _ifv_check(S, T, labels, classes_num)
    n, cs, h, w = S.shape
    ct, k = T.shape[1], int(classes_num)
    lab = labels_nearest(labels, h, w)
    loss = torch.empty((), device=S.device, dtype=torch.float32)
    PS = torch.empty((n, k, cs), device=S.device, dtype=torch.float32)
    stats = torch.empty((3, n, k), device=S.device, dtype=torch.float64)
    pix = torch.empty((3, n, h * w), device=S.device, dtype=torch.float32)
    ws = _ws(S.device, lib().skd_ifv_workspace(n, h * w, k, cs, ct))
    lib().skd_ifv_fwd(n, h * w, k, _p(lab), _p(S), cs, *_row_strides(S), _p(T), ct, *_row_strides(T), _p(loss), _p(PS), _p(stats),
                      _p(pix), _p(ws), _st())
    return loss, (lab, PS, stats, pix)


def ifv_bwd(S, saved, classes_num, grad_out):
    """d loss / d S of ifv_fwd (through the student's cosines and its prototypes) from its `saved` tensors, dense NHWC."""
    lab, PS, stats, pix = saved
    _f32(S)
    if S.dim() != 4 or tuple(lab.shape) != (S.shape[0],) + tuple(S.shape[2:]) or tuple(PS.shape) != (S.shape[0], classes_num, S.shape[1]):
        raise ValueError("intra-class variation: the saved tensors do not match the student map %s" % (tuple(S.shape),))
    if not 1 <= classes_num <= 255:
        raise ValueError("intra-class variation: the class count must be in [1, 255] (got %r)" % (classes_num,))
    n, cs, h, w = S.shape
    dS = empty_nhwc(n, cs, h, w, S.device)
    ws = _ws(S.device, lib().skd_ifv_workspace(n, h * w, classes_num, cs, cs))
    lib().skd_ifv_bwd(n, h * w, classes_num, _p(lab), _p(S), cs, *_row_strides(S), _p(PS), _p(stats), _p(pix), _p(grad_out), _p(dS),
                      *_row_strides(dS), _p(ws), _st())
    return dS


def _class_weight(weight, l0):
    """The class-weight table as the weighted kernels read it: contiguous fp32, one entry per class, on the logits' device."""
    if weight.dtype != torch.float32 or not weight.is_contiguous() or weight.dim() != 1 or weight.device != l0.device:
        raise ValueError("class weight must be a contiguous 1-D float32 tensor on the logits' device")
    if weight.numel() != l0.shape[1]:
        raise ValueError("class weight has %d entries for %d classes" % (weight.numel(), l0.shape[1]))
    return weight


def dsn_ce_fwd(l0, l1, labels, ignore_index, w0, w1, weight=None):
    """-> (loss, count): count is the number of valid pixels, or with `weight` (C class weights, fp32 on the device) the sum of their
    class weights."""
    _f32(l0, l1)
    n, c, h, w = l0.shape
    H, W = labels.shape[1:]
    if labels.dtype != torch.int64 or not labels.is_contiguous():
        raise ValueError("labels must be contiguous int64")
    out = torch.empty(2, device=l0.device, dtype=torch.float32)       # loss, valid count
    s1 = pixel_strides(l1) if l1 is not None else (0, 0, 0)
    args = (n, c, h, w, H, W, _p(l0), *pixel_strides(l0), _p(l1), *s1, _p(labels), ignore_index, w0, w1, _p(out[0]), _p(out[1]),
            _p(_ws(l0.device)))
    if weight is None:
        lib().skd_dsn_ce_fwd(*args, _st())
    else:
        lib().skd_dsn_ce_fwd_weighted(*args, _p(_class_weight(weight, l0)), _st())
    return out


def dsn_ce_fwd_train(l0, l1, labels, ignore_index, w0, w1, weight=None):
    """Training forward: (loss, count) tensor AND the backward's row-phase workspace, in one pass over the upsampled pixels.
    With `weight` the loss is class-weighted and count is the sum of the valid pixels' class weights (dsn_ce_bwd_cols divides by it)."""
    _f32(l0, l1)
    n, c, h, w = l0.shape
    H, W = labels.shape[1:]
    if labels.dtype != torch.int64 or not labels.is_contiguous():
        raise ValueError("labels must be contiguous int64")
    L = lib()
    heads = 2 if l1 is not None else 1
    out = torch.empty(2, device=l0.device, dtype=torch.float32)       # loss, valid count
    parts = torch.empty(L.skd_dsn_ce_train_partials(n, H, heads), device=l0.device, dtype=torch.float64)
    rows = torch.empty(L.skd_dsn_ce_bwd_workspace_floats(n, c, w, H, heads), device=l0.device, dtype=torch.float32)
    s1 = pixel_strides(l1) if l1 is not None else (0, 0, 0)
    args = (n, c, h, w, H, W, _p(l0), *pixel_strides(l0), _p(l1), *s1, _p(labels), ignore_index, w0, w1, _p(out[0]), _p(out[1]),
            _p(parts), _p(rows))
    if weight is None:
        L.skd_dsn_ce_fwd_train(*args, _st())
    else:
        L.skd_dsn_ce_fwd_train_weighted(*args, _p(_class_weight(weight, l0)), _st())
    return out, rows


def dsn_ce_bwd_cols(l0, l1, rows, H, w0, w1, grad_out, count):
    n, c, h, w = l0.shape
    d0 = torch.empty_strided(l0.shape, l0.stride(), device=l0.device, dtype=torch.float32)
    d1 = torch.empty_strided(l1.shape, l1.stride(), device=l1.device, dtype=torch.float32) if l1 is not None else None
    s1 = pixel_strides(l1) if l1 is not None else (0, 0, 0)
    lib().skd_dsn_ce_bwd_cols(n, c, h, w, H, _p(rows), *pixel_strides(l0), *s1, 2 if l1 is not None else 1, w0, w1, _p(grad_out), _p(count),
                              _p(d0), _p(d1), _st())
    return d0, d1


def ohem_grid_shape(H, W, factor):
    """Size of OhemCrossEntropy2d's threshold grid: scipy.ndimage.zoom's output shape, Python round(H * (1 / factor))
    (half to even: 36 / 8 -> 4, 44 / 8 -> 6)."""
    return int(round(H * (1.0 / factor))), int(round(W * (1.0 / factor)))


def ohem_grid_sample(logits, labels, factor, ignore_index, want_labels=False):
    """-> (pred (N, gh, gw) fp32 with +inf at ignored points, grid labels (N, gh, gw) int64 or None, valid count (1,) int32)."""
    _f32(logits)
    n, c, h, w = logits.shape
    H, W = labels.shape[1:]
    if labels.dtype != torch.int64 or not labels.is_contiguous():
        raise ValueError("labels must be contiguous int64")
    gh, gw = ohem_grid_shape(H, W, factor)
    pred = torch.empty((n, gh, gw), device=logits.device, dtype=torch.float32)
    glab = torch.empty((n, gh, gw), device=logits.device, dtype=torch.int64) if want_labels else None
    nvalid = torch.empty(1, device=logits.device, dtype=torch.int32)
    lib().skd_ohem_grid_sample(n, c, h, w, H, W, gh, gw, _p(logits), *pixel_strides(logits), _p(labels), ignore_index, _p(pred),
                               _p(glab), _p(nvalid), _st())
    return pred, glab, nvalid


def ohem_threshold(pred, nvalid, min_kept, thresh):
    """Device threshold (0-dim fp32) from the grid values: 1 if min_kept >= valid, else max(thresh, (min_kept-1)-th smallest)."""
    L = lib()
    ws = torch.empty(L.skd_ohem_threshold_workspace_ints(), device=pred.device, dtype=torch.int32)
    thr = torch.empty((), device=pred.device, dtype=torch.float32)
    L.skd_ohem_threshold(pred.numel(), _p(pred), _p(nvalid), int(min(min_kept, 2 ** 31 - 1)), float(thresh), _p(thr), _p(ws), _st())
    return thr


def ohem_dsn_ce_fwd_train(l0, l1, labels, ignore_index, w0, w1, threshold):
    """-> (loss 0-dim, counts (4,): kept, valid of head 1, backward denominators) and the backward's row-phase workspace."""
    _f32(l0, l1)
    n, c, h, w = l0.shape
    H, W = labels.shape[1:]
    if labels.dtype != torch.int64 or not labels.is_contiguous():
        raise ValueError("labels must be contiguous int64")
    L = lib()
    heads = 2 if l1 is not None else 1
    loss = torch.empty((), device=l0.device, dtype=torch.float32)
    counts = torch.empty(4, device=l0.device, dtype=torch.float32)
    parts = torch.empty(L.skd_dsn_ce_train_partials(n, H, heads), device=l0.device, dtype=torch.float64)
    rows = torch.empty(L.skd_dsn_ce_bwd_workspace_floats(n, c, w, H, heads), device=l0.device, dtype=torch.float32)
    s1 = pixel_strides(l1) if l1 is not None else (0, 0, 0)
    L.skd_ohem_dsn_ce_fwd_train(n, c, h, w, H, W, _p(l0), *pixel_strides(l0), _p(l1), *s1, _p(labels), ignore_index, w0, w1,
                                _p(threshold), _p(loss), _p(counts), _p(parts), _p(rows), _st())
    return loss, counts, rows


def ohem_dsn_ce_bwd_cols(l0, l1, rows, H, w0, w1, grad_out, counts):
    n, c, h, w = l0.shape
    d0 = torch.empty_strided(l0.shape, l0.stride(), device=l0.device, dtype=torch.float32)
    d1 = torch.empty_strided(l1.shape, l1.stride(), device=l1.device, dtype=torch.float32) if l1 is not None else None
    s1 = pixel_strides(l1) if l1 is not None else (0, 0, 0)
    lib().skd_ohem_dsn_ce_bwd_cols(n, c, h, w, H, _p(rows), *pixel_strides(l0), *s1, 2 if l1 is not None else 1, w0, w1, _p(grad_out),
                                   _p(counts), _p(d0), _p(d1), _st())
    return d0, d1


def dsn_ce_bwd(l0, l1, labels, ignore_index, w0, w1, grad_out, count):
    n, c, h, w = l0.shape
    H, W = labels.shape[1:]
    L = lib()
    heads = 2 if l1 is not None else 1
    ws = torch.empty(L.skd_dsn_ce_bwd_workspace_floats(n, c, w, H, heads), device=l0.device, dtype=torch.float32)
    # gradient tensors share the logits' strides exactly (pitched channel slices included)
    d0 = torch.empty_strided(l0.shape, l0.stride(), device=l0.device, dtype=torch.float32)
    d1 = torch.empty_strided(l1.shape, l1.stride(), device=l1.device, dtype=torch.float32) if l1 is not None else None
    s1 = pixel_strides(l1) if l1 is not None else (0, 0, 0)
    L.skd_dsn_ce_bwd(n, c, h, w, H, W, _p(l0), *pixel_strides(l0), _p(l1), *s1, _p(labels), ignore_index, w0, w1,
                     _p(grad_out), _p(count), _p(d0), _p(d1), _p(ws), _st())
    return d0, d1


def pairwise_pool(F, ph, pw, want_argmax):
    _f32(F)
    n, c, h, w = F.shape
    nh, nw = -(-h // ph), -(-w // pw)
    nodes = nh * nw
    pooled = torch.empty((n, nodes, c), device=F.device, dtype=torch.float32)
    arg = torch.empty((n, nodes, c), device=F.device, dtype=torch.int32) if want_argmax else None
    rnorm = torch.empty((n, nodes), device=F.device, dtype=torch.float32)
    lib().skd_pairwise_pool(n, c, h, w, _p(F), *pixel_strides(F), ph, pw, _p(pooled), _p(arg), _p(rnorm), _st())
    return pooled, arg, rnorm


def pairwise_gram(pS, pT, rS, rT, want_E):
    n, nodes, cs = pS.shape
    ct = pT.shape[2]
    L = lib()
    E = torch.empty((n, nodes, nodes), device=pS.device, dtype=torch.float32) if want_E else None
    loss = torch.empty((), device=pS.device, dtype=torch.float32)
    ws = _ws(pS.device, max(L.skd_pairwise_gram_partials(n, nodes), 8))
    L.skd_pairwise_gram(n, nodes, cs, ct, _p(pS), _p(pT), _p(rS), _p(rT), _p(E), _p(loss), _p(ws), _st())
    return loss, E


def pairwise_bwd(E, pS, rS, arg, grad_out, feat_like):
    n, nodes, cs = pS.shape
    dpooled = torch.empty_like(pS)
    dF = torch.zeros_like(feat_like)                 # keeps the feature's memory format
    lib().skd_pairwise_bwd(n, nodes, cs, _p(E), _p(pS), _p(rS), _p(arg), _p(grad_out), _p(dpooled), _p(dF),
                           *pixel_strides(dF), _st())
    return dF


def pairwise_affinity_sm100(pS, pT, rS, rT, want_E):
    """wgmma large-node path: loss (0-dim) and E (N, nodes, ldE) or None."""
    n, nodes, cs = pS.shape
    ct = pT.shape[2]
    L = lib()
    ldE = pad4(nodes)
    E = torch.empty((n, nodes, ldE), device=pS.device, dtype=torch.float32) if want_E else None
    ws = torch.empty(L.skd_pairwise_affinity_sm100_workspace_floats(n, nodes, cs, ct), device=pS.device, dtype=torch.float32)
    acc = torch.empty(1, device=pS.device, dtype=torch.float64)
    loss = torch.empty((), device=pS.device, dtype=torch.float32)
    L.skd_pairwise_affinity_sm100(n, nodes, cs, ct, _p(pS), _p(pT), _p(rS), _p(rT), _p(E), ldE, _p(loss), _p(ws), _p(acc), _st())
    return loss, E


def pairwise_affinity_bwd_sm100(E, pS, rS, arg, grad_out, feat_like):
    n, nodes, cs = pS.shape
    ldE = E.shape[2]
    L = lib()
    ws = torch.empty(L.skd_pairwise_affinity_bwd_sm100_workspace_floats(n, nodes, cs, ldE), device=pS.device, dtype=torch.float32)
    dpooled = torch.empty_like(pS)
    L.skd_pairwise_affinity_bwd_sm100(n, nodes, cs, _p(E), ldE, _p(pS), _p(rS), _p(grad_out), _p(dpooled), _p(ws), _st())
    dF = torch.zeros(feat_like.shape, device=feat_like.device, dtype=torch.float32).contiguous(memory_format=torch.channels_last) \
        if feat_like.dim() == 4 and feat_like.stride(1) == 1 else torch.zeros_like(feat_like)
    L.skd_pairwise_scatter(n, nodes, cs, _p(dpooled), _p(arg), _p(dF), *pixel_strides(dF), _st())
    return dF


def pairwise_local_pairs(h, w, k, d):
    """Connected ordered pairs per image of the local pair-wise term on an h x w node grid (window k, dilation d)."""
    return int(lib().skd_pairwise_local_pairs(h, w, k, d))


def pairwise_local_fwd(pS, pT, rS, rT, h, w, k, d, want_E):
    """Local pair-wise term over pairwise_pool's rows on their h x w node grid (csrc/pairwise_local.cu): loss (0-dim) and
    E (N, h*w, k*k) or None."""
    n, nodes, cs = pS.shape
    ct = pT.shape[2]
    if nodes != h * w or pT.shape[:2] != pS.shape[:2]:
        raise ValueError("local pair-wise: pooled rows %s / %s do not cover a %dx%d grid" % (tuple(pS.shape), tuple(pT.shape), h, w))
    L = lib()
    E = torch.empty((n, nodes, k * k), device=pS.device, dtype=torch.float32) if want_E else None
    parts = torch.empty(L.skd_pairwise_local_partials(n, h, w, k, d), device=pS.device, dtype=torch.float64)
    loss = torch.empty((), device=pS.device, dtype=torch.float32)
    L.skd_pairwise_local_fwd(n, h, w, cs, ct, _p(pS), _p(pT), _p(rS), _p(rT), k, d, _p(E), _p(loss), _p(parts), _st())
    return loss, E


def pairwise_local_bwd(E, pS, rS, h, w, k, d, arg, grad_out, feat_like):
    """d loss / d feature of pairwise_local_fwd: the pooled rows' gradient, scattered through the max-pool argmax (in feat_like's
    layout, channels-last when feat_like is)."""
    n, nodes, cs = pS.shape
    dpooled = torch.empty_like(pS)
    L = lib()
    L.skd_pairwise_local_bwd(n, h, w, cs, _p(E), _p(pS), _p(rS), k, d, _p(grad_out), _p(dpooled), _st())
    dF = torch.zeros(feat_like.shape, device=feat_like.device, dtype=torch.float32).contiguous(memory_format=torch.channels_last) \
        if feat_like.dim() == 4 and feat_like.stride(1) == 1 else torch.zeros_like(feat_like)
    L.skd_pairwise_scatter(n, nodes, cs, _p(dpooled), _p(arg), _p(dF), *pixel_strides(dF), _st())
    return dF


# ------------------------------------------------------------------------------------------------ ESPNet-C (csrc/espnet.cu)
def _rows(t):
    """-> (P, C, pitch) of an NHWC-stored (possibly channel-sliced) tensor."""
    n, c, h, w, pitch = nhwc_meta(t)
    return n * h * w, c, pitch


def bnprelu_stats(x, momentum, running_mean, running_var, num_batches_tracked):
    """Batch mean / biased variance of x's channels; running statistics and the batch counter updated in place (may be None)."""
    _f32(x)
    P, c, ldx = _rows(x)
    st = torch.empty(2, c, device=x.device)
    ws = torch.empty(lib().skd_bnprelu_workspace_doubles(P, c), device=x.device, dtype=torch.float64)
    lib().skd_bnprelu_stats(P, c, _p(x), ldx, momentum, _p(running_mean), _p(running_var), _p(num_batches_tracked), _p(st[0]), _p(st[1]),
                            _p(ws), _st())
    return st


def esp_combine(branches, residual, out, momentum=0.0, running_mean=None, running_var=None, num_batches_tracked=None, stats=True):
    """ESP combine of the five branch outputs (d1, d2, d4, d8, d16: NHWC tensors, channel-padded) plus the optional residual into `out`
    ((N, n1 + 4n, H, W) NHWC); -> batch statistics (2, C) or None."""
    d1, d2, d4, d8, d16 = branches
    P, n1, ld1 = _rows(d1)
    _, n, ldn = _rows(d2)
    for t in (d4, d8, d16):
        if _rows(t)[2] != ldn:
            raise ValueError("Non-contiguous input")
    _, c, ldo = _rows(out)
    ldr = _rows(residual)[2] if residual is not None else 0
    L = lib()
    st = torch.empty(2, c, device=out.device) if stats else None
    ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, c), device=out.device, dtype=torch.float64) if stats else None
    L.skd_esp_combine(P, n1, n, _p(d1), ld1, _p(d2), _p(d4), _p(d8), _p(d16), ldn, _p(residual), ldr, _p(out), ldo, momentum,
                      _p(running_mean), _p(running_var), _p(num_batches_tracked), _p(st[0]) if stats else None,
                      _p(st[1]) if stats else None, _p(ws), _st())
    return st


def bnprelu_apply(x, mean, var, weight, bias, alpha, eps, out=None, out_channels=None):
    """prelu(bn(x)) -> `out` (default: a fresh NHWC tensor with `out_channels` >= C channels, the extra ones zero).  alpha=None: bn(x)
    alone (here and in the two backward passes)."""
    _f32(x)
    n, c, h, w, ldx = nhwc_meta(x)
    cw = out_channels or c
    if out is None:
        out = empty_nhwc(n, cw, h, w, x.device)
    ldo = nhwc_meta(out)[4]
    lib().skd_bnprelu_apply(n * h * w, c, _p(x), ldx, _p(mean), _p(var), _p(weight), _p(bias), _p(alpha), eps, _p(out), ldo, cw, _st())
    return out


def bnprelu_bwd_reduce(x, dout, mean, var, weight, bias, alpha, eps):
    """-> (dweight, dbias, dalpha) and the (2, C) coefficients of the dx pass."""
    P, c, ldx = _rows(x)
    ldd = _rows(dout)[2]
    L = lib()
    red = torch.empty(5, c, device=x.device)             # dweight, dbias, dalpha, mean dz, mean dz*xhat
    ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, c), device=x.device, dtype=torch.float64)
    L.skd_bnprelu_bwd_reduce(P, c, _p(x), ldx, _p(dout), ldd, _p(mean), _p(var), _p(weight), _p(bias), _p(alpha), eps, _p(red[0]),
                             _p(red[1]), _p(red[2]) if alpha is not None else None, _p(red[3]), _p(ws), _st())
    return red[0], red[1], red[2] if alpha is not None else None, red[3:5]


def bnprelu_bwd_dx(x, dout, mean, var, weight, bias, alpha, eps, training, coef, dx_channels=None):
    n, c, h, w, ldx = nhwc_meta(x)
    ldd = nhwc_meta(dout)[4]
    cw = dx_channels or c
    dx = empty_nhwc(n, cw, h, w, x.device)
    lib().skd_bnprelu_bwd_dx(n * h * w, c, _p(x), ldx, _p(dout), ldd, _p(mean), _p(var), _p(weight), _p(bias), _p(alpha), eps,
                             int(training), _p(coef), _p(dx), cw, cw, _st())
    return dx


def esp_bwd_dx(x, dout, mean, var, weight, bias, alpha, eps, training, coef, n1, n, want_dres):
    """-> (dd1, dd2, dd4, dd8, dd16) (channel-padded to multiples of 4, pad channels zero) and dres (or None)."""
    N, c, h, w, ldx = nhwc_meta(x)
    ldd = nhwc_meta(dout)[4]
    dev = x.device
    dd1 = empty_nhwc(N, pad4(n1), h, w, dev)
    dds = [empty_nhwc(N, pad4(n), h, w, dev) for _ in range(4)]
    dres = empty_nhwc(N, c, h, w, dev) if want_dres else None
    lib().skd_esp_bwd_dx(N * h * w, n1, n, _p(x), ldx, _p(dout), ldd, _p(mean), _p(var), _p(weight), _p(bias), _p(alpha), eps,
                         int(training), _p(coef), _p(dd1), pad4(n1), *[_p(t) for t in dds], pad4(n), _p(dres), c, _st())
    return (dd1, *dds), dres


def resample_adjoint_nhwc(dout, h, w, channels=None):
    """Adjoint of resample_nhwc(t, H, W) for t of size (h, w): (N, C, H, W) gradient -> (N, C, h, w) NHWC gradient, padded to
    `channels` >= C (pad channels zero).  Fixed-order gather, bit-identical across calls."""
    _f32(dout)
    dout = dout.contiguous(memory_format=torch.channels_last)
    n, c, H, W = dout.shape
    cw = channels or c
    dsrc = (torch.zeros if cw != c else torch.empty)((n, h, w, cw), device=dout.device, dtype=torch.float32)
    lib().skd_resample_bilinear_adjoint_nhwc(n, c, h, w, _p(dout), H, W, _p(dsrc), cw, _st())
    return dsrc.permute(0, 3, 1, 2)


def avgpool3x3s2(src, out):
    """nn.AvgPool2d(3, 2, 1) of src (N, C, H, W) NHWC(-pitched) into out (N, C, (H+1)//2, (W+1)//2) NHWC(-pitched), in place."""
    n, c, h, w, lds = nhwc_meta(src)
    ldd = nhwc_meta(out)[4]
    lib().skd_avgpool3x3s2(n, h, w, c, _p(src), lds, _p(out), ldd, _st())
    return out


def resample_nhwc(t, h, w):
    """Bilinear (align_corners=True) resize of an (N, C, H', W') tensor to (N, C, h, w), NHWC output; forward only."""
    _f32(t)
    n, c = t.shape[:2]
    out = torch.empty((n, h, w, c), device=t.device, dtype=torch.float32)
    lib().skd_resample_bilinear_nhwc(n, c, t.shape[2], t.shape[3], _p(t), *pixel_strides(t), h, w, _p(out), _st())
    return out.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ MobileNetV2 (csrc/mobilenet.cu)
def dwconv_check(channels, weight_shape, stride, dilation):
    """ValueError unless the depthwise shape is one the kernels run: a (C, 1, 3, 3) weight, C a multiple of 4, stride 1 or 2,
    dilation >= 1 (padding = dilation)."""
    if tuple(weight_shape) != (channels, 1, 3, 3):
        raise ValueError("depthwise conv: weight must be (C, 1, 3, 3) = (%d, 1, 3, 3), got %s" % (channels, tuple(weight_shape)))
    if channels % 4:
        raise ValueError("depthwise conv: C must be a multiple of 4 (got %d)" % channels)
    if stride not in (1, 2) or int(dilation) < 1:
        raise ValueError("depthwise conv: stride must be 1 or 2 and dilation >= 1 (got stride %r, dilation %r)" % (stride, dilation))


def dense_nhwc(t):
    t = to_nhwc(t)
    if nhwc_meta(t)[4] != t.shape[1]:
        t = t.contiguous(memory_format=torch.channels_last)
    return t


def _mbv2_ws(P, c, device):
    return torch.empty(max(int(lib().skd_mbv2_workspace_doubles(P, c)), 1), device=device, dtype=torch.float64)


def dwconv3x3_fwd(x, weight, stride, dilation, stats=False, momentum=0.0, running_mean=None, running_var=None, num_batches_tracked=None):
    """Depthwise 3x3 convolution (padding = dilation) of an (N, C, H, W) tensor -> (dense NHWC output, its (2, C) batch statistics or
    None).  With `stats` the BatchNorm that follows gets its mean / biased variance (and its running statistics) from the same pass."""
    n, c, h, w = x.shape
    dwconv_check(c, weight.shape, stride, dilation)
    _f32(x, weight)
    x = dense_nhwc(x)
    oh, ow = (h - 1) // stride + 1, (w - 1) // stride + 1
    y = empty_nhwc(n, c, oh, ow, x.device)
    st = torch.empty(2, c, device=x.device) if stats else None
    ws = _mbv2_ws(n * oh * ow, c, x.device) if stats else None
    lib().skd_dwconv3x3_fwd(n, h, w, c, stride, int(dilation), _p(x), _p(weight.contiguous()), _p(y), momentum, _p(running_mean),
                            _p(running_var), _p(num_batches_tracked), _p(st[0]) if stats else None, _p(st[1]) if stats else None,
                            _p(ws), _st())
    return y, st


def dwconv3x3_dgrad(dy, weight, x_shape, stride, dilation):
    n, c, h, w = x_shape
    dwconv_check(c, weight.shape, stride, dilation)
    _f32(dy, weight)
    dy = dense_nhwc(dy)
    dx = empty_nhwc(n, c, h, w, dy.device)
    lib().skd_dwconv3x3_dgrad(n, h, w, c, stride, int(dilation), _p(dy), _p(weight.contiguous()), _p(dx), _st())
    return dx


def dwconv3x3_wgrad(x, dy, stride, dilation):
    """-> the (C, 1, 3, 3) weight gradient (fixed-order reduction over every output pixel)."""
    n, c, h, w = x.shape
    dwconv_check(c, (c, 1, 3, 3), stride, dilation)
    _f32(x, dy)
    x, dy = dense_nhwc(x), dense_nhwc(dy)
    dw = torch.empty((c, 1, 3, 3), device=x.device, dtype=torch.float32)
    ws = _mbv2_ws(n * dy.shape[2] * dy.shape[3], c, x.device)
    lib().skd_dwconv3x3_wgrad(n, h, w, c, stride, int(dilation), _p(x), _p(dy), _p(dw), _p(ws), _st())
    return dw


def bnact_apply(x, mean, var, weight, bias, eps, relu6, residual=None):
    """relu6(bn(x)) (relu6=True) or bn(x) + residual (relu6=False; residual may be None) -> fresh dense NHWC tensor."""
    _f32(x, residual)
    P, c, ldx = _rows(x)
    out = empty_nhwc(x.shape[0], c, x.shape[2], x.shape[3], x.device)
    ldr = _rows(residual)[2] if residual is not None else 0
    lib().skd_bnact_apply(P, c, int(relu6), _p(x), ldx, _p(mean), _p(var), _p(weight), _p(bias), eps, _p(residual), ldr, _p(out), c,
                          _st())
    return out


def bnact_bwd_reduce(x, dout, mean, var, weight, bias, eps, relu6):
    """-> (dweight, dbias) and the (2, C) coefficients of the dx pass."""
    P, c, ldx = _rows(x)
    ldd = _rows(dout)[2]
    red = torch.empty(4, c, device=x.device)             # dweight, dbias, mean dz, mean dz*xhat
    lib().skd_bnact_bwd_reduce(P, c, int(relu6), _p(x), ldx, _p(dout), ldd, _p(mean), _p(var), _p(weight), _p(bias), eps, _p(red[0]),
                               _p(red[1]), _p(red[2]), _p(_mbv2_ws(P, c, x.device)), _st())
    return red[0], red[1], red[2:4]


def bnact_bwd_dx(x, dout, mean, var, weight, bias, eps, relu6, training, coef):
    P, c, ldx = _rows(x)
    ldd = _rows(dout)[2]
    dx = empty_nhwc(x.shape[0], c, x.shape[2], x.shape[3], x.device)
    lib().skd_bnact_bwd_dx(P, c, int(relu6), _p(x), ldx, _p(dout), ldd, _p(mean), _p(var), _p(weight), _p(bias), eps, int(training),
                           _p(coef), _p(dx), c, _st())
    return dx


def sgd_step_nvls(lo, hi, param_mc, grad_mc, param_local, buf, lr_dev, momentum, weight_decay, grad_scale):
    """data-parallel SGD over NVSwitch multicast on the owned range [lo, hi): see include/skd.h skd_sgd_step_nvls"""
    lib().skd_sgd_step_nvls(int(lo), int(hi), int(param_mc), int(grad_mc), _p(param_local), _p(buf), _p(lr_dev), momentum, weight_decay,
                            grad_scale, _st())


def sgd_step(param, grad, buf, lr_dev, momentum, weight_decay, first, grad_scale=1.0):
    lib().skd_sgd_step(param.numel(), _p(param), _p(grad), _p(buf), _p(lr_dev), momentum, weight_decay, int(first), grad_scale, _st())
