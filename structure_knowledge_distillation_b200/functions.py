"""torch.autograd.Functions over the sm_90a kernels (the reference's libs/functions.py role, for the whole hot path).

Conventions kept from the reference (libs/functions.py:70-162): ctx.save_for_backward for tensors, non-tensor
arguments get None gradients, backward is once-differentiable (no double backward through hand-written kernels).
"""
import torch
import torch.distributed as dist
from torch.autograd.function import once_differentiable

from . import ops


# ------------------------------------------------------------------------------------------------ losses
class PixelWiseLoss(torch.autograd.Function):
    """CriterionPixelWise math (utils/criterion.py:219-226) in one warp-reduced kernel each way."""

    @staticmethod
    def forward(ctx, logits_S, logits_T):
        ctx.save_for_backward(logits_S, logits_T)
        return ops.pixelwise_fwd(logits_S, logits_T)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        S, T = ctx.saved_tensors
        return ops.pixelwise_bwd(S, T, g.contiguous()), None


class PairWiseLoss(torch.autograd.Function):
    """CriterionPairWiseforWholeFeatAfterPool math (utils/criterion.py:236-245, utils/utils.py:170-183)."""

    TCGEN05_MIN_NODES = 1024      # below: one SIMT tile kernel (the default pool_scale 0.5 has 9 nodes); above: wgmma GEMM

    @staticmethod
    def forward(ctx, feat_S, feat_T, ph, pw):
        pS, arg, rS = ops.pairwise_pool(feat_S, ph, pw, True)
        pT, _, rT = ops.pairwise_pool(feat_T, ph, pw, False)
        ctx.tensor_core = pS.shape[1] >= PairWiseLoss.TCGEN05_MIN_NODES and (pS.shape[2] + pT.shape[2]) % 4 == 0 and pS.shape[2] % 4 == 0
        need_E = feat_S.requires_grad
        if ctx.tensor_core:
            loss, E = ops.pairwise_affinity_sm100(pS, pT, rS, rT, need_E)
        else:
            loss, E = ops.pairwise_gram(pS, pT, rS, rT, True)
        ctx.save_for_backward(E, pS, rS, arg, feat_S)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        E, pS, rS, arg, feat_S = ctx.saved_tensors
        if ctx.tensor_core:
            return ops.pairwise_affinity_bwd_sm100(E, pS, rS, arg, g.contiguous(), feat_S), None, None, None
        return ops.pairwise_bwd(E, pS, rS, arg, g.contiguous(), feat_S), None, None, None


class PairWiseLocalLoss(torch.autograd.Function):
    """The pair-wise term with each pooled node connected to its `window` x `window` neighbours at `dilation` (the pooled grid's
    nodes j = (y + t d, x + u d) inside the grid, t, u in -r..r): sum over those pairs of (a^T_ij - a^S_ij)^2 / (N * P), P the connected
    pairs per image.  Pooling and the detached norm are PairWiseLoss's; E is (N, nodes, window^2), never nodes^2."""

    @staticmethod
    def forward(ctx, feat_S, feat_T, ph, pw, window, dilation):
        pS, arg, rS = ops.pairwise_pool(feat_S, ph, pw, True)
        pT, _, rT = ops.pairwise_pool(feat_T, ph, pw, False)
        h, w = -(-feat_S.shape[2] // ph), -(-feat_S.shape[3] // pw)
        loss, E = ops.pairwise_local_fwd(pS, pT, rS, rT, h, w, window, dilation, feat_S.requires_grad)
        ctx.grid = (h, w, window, dilation)
        ctx.save_for_backward(E, pS, rS, arg, feat_S)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        E, pS, rS, arg, feat_S = ctx.saved_tensors
        return ops.pairwise_local_bwd(E, pS, rS, *ctx.grid, arg, g.contiguous(), feat_S), None, None, None, None, None


class AttentionTransferLoss(torch.autograd.Function):
    """Attention transfer (Zagoruyko & Komodakis): mean over N*H*W of (at(S) - at(T))^2 with at(x) = F.normalize(x.pow(2).mean(1)
    .view(N, -1)).  The forward keeps the normalised maps and the student's norms for the backward; the teacher gets no gradient."""

    @staticmethod
    def forward(ctx, feat_S, feat_T):
        loss, qhat, norms = ops.at_fwd(feat_S, feat_T)
        ctx.save_for_backward(feat_S, qhat, norms)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        feat_S, qhat, norms = ctx.saved_tensors
        return ops.at_bwd(feat_S, qhat, norms, g.contiguous()), None


class MseLoss(torch.autograd.Function):
    """F.mse_loss(r, t) with t frozen: MIMIC's regression of the teacher's feature map from the adapter output r."""

    @staticmethod
    def forward(ctx, r, t):
        ctx.save_for_backward(r, t)
        return ops.mse_fwd(r, t)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        r, t = ctx.saved_tensors
        return ops.mse_bwd(r, t, g.contiguous()), None


class ChannelWiseLoss(torch.autograd.Function):
    """Channel-wise distillation (Shu et al.): tau^2 / (N*C) * sum over (n, c) of KL(pT || pS), p the softmax of x / tau over the H*W
    positions of each channel, S and T of one shape.  log p is computed as x / tau - logsumexp (max-subtracted), not as
    softmax(...).log(): the two agree wherever pS does not underflow, and where it does this form stays finite while the other gives
    inf / NaN.  The forward keeps the per-channel log-sum-exps; the backward recomputes both softmaxes from them, so no probability
    map is stored.  The teacher gets no gradient."""

    @staticmethod
    def forward(ctx, feat_S, feat_T, tau):
        loss, lse = ops.cwd_fwd(feat_S, feat_T, tau)
        ctx.save_for_backward(feat_S, feat_T, lse)
        ctx.tau = tau
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        feat_S, feat_T, lse = ctx.saved_tensors
        return ops.cwd_bwd(feat_S, feat_T, lse, ctx.tau, g.contiguous()), None, None


class IntraClassVariationLoss(torch.autograd.Function):
    """Intra-class feature variation distillation (Wang et al., IFVD): per image and class k in [0, K), the prototype of each map is the
    mean feature of the pixels labelled k (the labels taken down to the maps' grid by nearest, / (count + 1e-6)); the loss is the mean
    over all N*h*w pixels of (cos(f_S, P_S) - cos(f_T, P_T))^2, cos torch's cosine_similarity (eps 1e-8).  A pixel labelled outside
    [0, K) (the ignore label) adds exactly 0 to the loss and the gradient; IFVD's code makes it its own centre, cos = 1 in both maps, which
    agrees up to the last bits.  S gets its gradient through its cosines and through its prototypes; the teacher gets none.  S and T may
    differ in width."""

    @staticmethod
    def forward(ctx, feat_S, feat_T, labels, classes_num):
        loss, saved = ops.ifv_fwd(feat_S, feat_T, labels, classes_num)
        ctx.save_for_backward(feat_S, *saved)
        ctx.classes_num = classes_num
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        feat_S, *saved = ctx.saved_tensors
        return ops.ifv_bwd(feat_S, saved, ctx.classes_num, g.contiguous()), None, None, None


class DsnCrossEntropy(torch.autograd.Function):
    """CriterionDSN math (utils/criterion.py:179-188): fused upsample + log-softmax + NLL for both heads.  `weight` (C fp32 class
    weights on the device, or None) makes each head's term CrossEntropyLoss(weight=weight)'s weighted mean."""

    @staticmethod
    def forward(ctx, l0, l1, labels, ignore_index, w0, w1, weight=None):
        # with a backward to come, the forward pass over the upsampled pixels already leaves the backward's row-phase result behind
        # (one softmax per pixel and step instead of two); inference keeps the plain forward
        ctx.fused = l0.requires_grad or (l1 is not None and l1.requires_grad)
        if ctx.fused:
            out, rows = ops.dsn_ce_fwd_train(l0, l1, labels, ignore_index, w0, w1, weight)
            ctx.save_for_backward(l0, l1, rows, out)
            ctx.H = labels.shape[1]
        else:
            # (no backward can follow: the weighted form needs no unfused backward)
            out = ops.dsn_ce_fwd(l0, l1, labels, ignore_index, w0, w1, weight)
            ctx.save_for_backward(l0, l1, labels, out)
        ctx.cfg = (ignore_index, w0, w1)
        return out[0].clone()

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        ig, w0, w1 = ctx.cfg
        if ctx.fused:
            l0, l1, rows, out = ctx.saved_tensors
            d0, d1 = ops.dsn_ce_bwd_cols(l0, l1, rows, ctx.H, w0, w1, g.contiguous(), out[1])
        else:
            l0, l1, labels, out = ctx.saved_tensors
            d0, d1 = ops.dsn_ce_bwd(l0, l1, labels, ig, w0, w1, g.contiguous(), out[1])
        return d0, d1, None, None, None, None, None


class OhemDsnCrossEntropy(torch.autograd.Function):
    """OhemCrossEntropy2d (utils/criterion.py:11-90) on head 0, plain CE on head 1 (l1 may be None), as CriterionOhemDSN
    (:200-209) combines them: w0 * OHEM-CE(up(l0)) + w1 * CE(up(l1)).  The threshold pass (1/factor grid + exact radix select)
    and the masked cross entropy run on the device, so there is no host sync.  Returns (loss, threshold, kept count); only the
    loss carries a gradient."""

    @staticmethod
    def forward(ctx, l0, l1, labels, ignore_index, thresh, min_kept, factor, w0, w1):
        pred, _, nvalid = ops.ohem_grid_sample(l0, labels, factor, ignore_index)
        thr = ops.ohem_threshold(pred, nvalid, min_kept // (factor * factor), thresh)
        loss, counts, rows = ops.ohem_dsn_ce_fwd_train(l0, l1, labels, ignore_index, w0, w1, thr)
        ctx.save_for_backward(l0, l1, rows, counts)
        ctx.cfg = (labels.shape[1], w0, w1)
        kept = counts[0].clone()
        ctx.mark_non_differentiable(thr, kept)
        return loss, thr, kept

    @staticmethod
    @once_differentiable
    def backward(ctx, g, g_thr, g_kept):
        l0, l1, rows, counts = ctx.saved_tensors
        H, w0, w1 = ctx.cfg
        d0, d1 = ops.ohem_dsn_ce_bwd_cols(l0, l1, rows, H, w0, w1, g.contiguous(), counts)
        return d0, d1, None, None, None, None, None, None, None


# ------------------------------------------------------------------------------------------------ layers
def _padded_weight(w_ohwi, cout_p, cin_p):
    cout, kh, kw, cin = w_ohwi.shape
    if cout_p == cout and cin_p == cin:
        return w_ohwi
    wp = torch.zeros((cout_p, kh, kw, cin_p), device=w_ohwi.device, dtype=torch.float32)
    wp[:cout, :, :, :cin] = w_ohwi
    return wp


def conv_forward_padded(x, weight, bias, stride, pad, dil, **epi):
    """wgmma forward for any channel count: Cin / Cout that are not multiples of 4 (3-channel image, 19 classes) are
    zero-padded to the next multiple so that every pixel row is 16-byte aligned for TMA.  Returns a (N,Cout,OH,OW) view."""
    w = ops.weight_ohwi(weight)
    cout, kh, kw, cin = w.shape
    cin_p, cout_p = ops.pad4(cin), ops.pad4(cout)
    if x.shape[1] != cin_p:                                   # callers may hand in an already padded image
        x = ops.pad_channels(x, cin_p)
    wp = _padded_weight(w, cout_p, cin_p)
    if cout_p != cout:
        for k in ("scale", "shift"):
            v = epi.get(k)
            if v is not None:
                pv = torch.zeros(cout_p, device=v.device, dtype=torch.float32); pv[:cout] = v; epi[k] = pv
        if bias is not None:
            pb = torch.zeros(cout_p, device=bias.device, dtype=torch.float32); pb[:cout] = bias; bias = pb
    if bias is not None:
        sc = epi.get("scale")
        epi["shift"] = bias if epi.get("shift") is None else epi["shift"] + (bias * sc if sc is not None else bias)
    y = ops.conv2d_fwd(x, wp, stride, pad, dil, **epi)
    return y[:, :cout] if cout_p != cout else y, x


def _small_cin(weight):
    return weight.shape[1] <= 4 and weight.shape[2] * weight.shape[3] > 1


def conv_forward_small_cin(x, weight, stride, pad, dil, precise=False, **epi):
    """Tiny-Cin convolution (3-channel stem) as explicit im2col + one dense K=32 GEMM step on wgmma."""
    cout, cin, kh, kw = weight.shape
    k = kh * kw * cin
    kp = (k + 31) // 32 * 32
    xin = x[:, :cin] if x.shape[1] != cin else x
    col = ops.im2col_small(xin, kh, kw, stride, pad, dil, kp)
    wp = torch.zeros((cout, 1, 1, kp), device=weight.device, dtype=torch.float32)
    wp[:, 0, 0, :k] = ops.weight_ohwi(weight).reshape(cout, k)
    if precise:
        return ops.conv2d_fwd_3xtf32(col, wp, 1, 0, 1), col
    return ops.conv2d_fwd(col, wp, 1, 0, 1, **epi), col


def _direct_grad(param, shape_ohwi=None):
    """The parameter's view of FlatSGD's gradient buffer when the optimizer asked for direct gradient writes (optim.FlatSGD,
    direct_grads=True) and its memory is the dense OHWI / 1-D layout the kernels produce; else None."""
    g = getattr(param, "_skd_grad", None)
    if g is None:
        return None
    if shape_ohwi is not None:
        cout, kh, kw, cin = shape_ohwi
        dense = (kh * kw * cin, 1, kw * cin, cin)                # the stride of a size-1 dimension does not matter (1x1 filters)
        if tuple(g.shape) != (cout, cin, kh, kw) or any(n > 1 and s != d for n, s, d in zip(g.shape, g.stride(), dense)):
            return None
    elif g.dim() != 1 or not g.is_contiguous():
        return None
    return g


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _sync_mean(t):
    dist.all_reduce(t)
    t /= _world()


class WgradOverlap:
    """Weight-gradient kernels on a side stream.  In the backward pass only the data-gradient chain (dgrad -> ABN backward -> dgrad
    ...) is sequential; a layer's weight gradient needs (x, dy) and feeds nothing but the optimizer.  Issued on a second stream the
    wgmma wgrad kernels overlap the HBM-bound ABN backward passes of the chain instead of queueing between them.  A wgrad CTA
    (384 threads, 39-58 K registers, 93-177 KB of shared memory) does not fit on an SM beside a large forward / data-gradient
    conv CTA (about 200 KB of shared memory), so it overlaps the small ABN kernels, not those convolutions.  NetModel opens a window around G_loss.backward(); tensors a side-stream kernel reads are kept alive
    until the window's join, so the caching allocator cannot hand their memory to a main-stream kernel early (valid in eager
    mode and under CUDA-graph capture alike -- no record_stream)."""
    stream = None
    keep = None

    @classmethod
    def begin(cls):
        if cls.stream is None:
            cls.stream = torch.cuda.Stream()
        cls.keep = []

    @classmethod
    def end(cls):
        if cls.keep is None:
            return
        torch.cuda.current_stream().wait_stream(cls.stream)
        cls.keep = None

    @classmethod
    def run(cls, fn, *tensors):
        """fn() on the side stream after everything enqueued so far on the current stream (no-op wrapper outside a window)."""
        if cls.keep is None:
            return fn()
        cls.stream.wait_stream(torch.cuda.current_stream())
        cls.keep.extend(t for t in tensors if t is not None)
        with torch.cuda.stream(cls.stream):
            out = fn()
        if isinstance(out, torch.Tensor):
            cls.keep.append(out)
        return out


def _grad_written(param):
    cb = getattr(param, "_skd_arrived", None)          # bucketed all-reduce bookkeeping (optim.FlatSGD.enable_overlap)
    if cb is not None:
        cb()


class Conv2d(torch.autograd.Function):
    """nn.Conv2d forward / dgrad / wgrad on wgmma.  x is NHWC-stored; weight is the (Cout,Cin,KH,KW) parameter held in
    channels-last (OHWI) storage."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, pad, dil, precise=False):
        ctx.small = _small_cin(weight) and bias is None and not x.requires_grad
        if ctx.small:
            y, xin = conv_forward_small_cin(x, weight, stride, pad, dil, precise=precise)
        elif precise and weight.shape[0] % 4 == 0 and weight.shape[1] % 4 == 0 and ops.nhwc_meta(x)[4] == x.shape[1]:
            # split-precision (3xTF32) forward for the layers whose rounding error train-mode BN amplifies most
            xin = x
            y = ops.conv2d_fwd_3xtf32(x, ops.weight_ohwi(weight), stride, pad, dil, shift=bias)
        else:
            y, xin = conv_forward_padded(x, weight, bias, stride, pad, dil)
        ctx.save_for_backward(xin, weight)
        ctx.params = (weight, bias)                          # the Parameter objects (their flat gradient views hang on them)
        ctx.cfg = (stride, pad, dil, bias is not None, tuple(x.shape))
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        xin, weight = ctx.saved_tensors
        stride, pad, dil, has_bias, xshape = ctx.cfg
        w = ops.weight_ohwi(weight)
        cout, kh, kw, cin = w.shape
        if ctx.small:                                        # xin is the im2col matrix: the weight gradient is a single-tap GEMM
            dwc = ops.conv2d_wgrad(xin, ops.to_nhwc(dy), (1, 1), 1, 0, 1)               # [Cout][1][1][Kp] (main stream: its result is reshaped right here)
            dw = dwc.reshape(cout, -1)[:, :kh * kw * cin].reshape(cout, kh, kw, cin).permute(0, 3, 1, 2)
            return None, dw, None, None, None, None, None
        cin_p, cout_p = ops.pad4(cin), ops.pad4(cout)
        dy = ops.pad_channels(dy, cout_p) if cout_p != cout else ops.to_nhwc(dy)
        if ops.nhwc_meta(dy)[4] % 4:
            dy = ops.pad_channels(dy, cout_p)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            wp = _padded_weight(w, cout_p, cin_p)
            dx = ops.conv2d_dgrad(dy, wp, (xshape[0], cin_p, xshape[2], xshape[3]), stride, pad, dil)
            if cin_p != cin:
                dx = dx[:, :cin]
        wparam, bparam = ctx.params
        if ctx.needs_input_grad[1]:
            gview = _direct_grad(wparam, (cout, kh, kw, cin)) if (cout_p == cout and cin_p == cin) else None
            if gview is not None:                            # wgrad (and its split-K reduction) writes the flat gradient buffer itself
                WgradOverlap.run(lambda: ops.conv2d_wgrad(xin, dy, (kh, kw), stride, pad, dil, out=gview), xin, dy)
                _grad_written(wparam)
            else:
                dw = ops.conv2d_wgrad(xin, dy, (kh, kw), stride, pad, dil)
                dw = dw[:cout, :, :, :cin].permute(0, 3, 1, 2)
        if has_bias and ctx.needs_input_grad[2]:
            gview = _direct_grad(bparam) if cout_p == cout else None
            if gview is not None:
                ops.colsum(dy, out=gview)
                _grad_written(bparam)
            else:
                db = ops.colsum(dy)[:cout]
        return dx, dw, db, None, None, None, None


class ABN(torch.autograd.Function):
    """InPlaceABN(Sync) forward/backward (libs/functions.py:70-162) fused with what follows it in the network:
    the ReLU the backbone applies right after an activation='none' ABN (networks/pspnet_combine.py:36,69,177), the
    residual add + ReLU that closes a block (:42-43,81-82) and the Dropout2d after the PSP / DSN ABN (:99,143)."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, training, momentum, eps, activation, slope, residual,
                chan_mul, sync=False):
        ctx.sync = bool(sync) and training and _world() > 1
        if ctx.sync:
            # InPlaceABNSync across processes (libs/functions.py:177-209): per-rank mean / biased variance, combined as
            # mean = E[mean_r], var = E[var_r + (mean - mean_r)^2] (equal per-rank counts, like the reference), running statistics
            # with the GLOBAL sample count; one small all-reduce per layer and direction
            loc = ops.abn_stats(x, weight, bias, eps, momentum, None, None)
            m = torch.stack([loc[0], loc[1] + loc[0] * loc[0]])
            dist.all_reduce(m)
            m /= _world()
            mean, var = m[0], (m[1] - m[0] * m[0]).clamp_min_(0)
            n = float(x.numel() // x.shape[1]) * _world()
            running_mean.mul_(1 - momentum).add_(mean, alpha=momentum)
            running_var.mul_(1 - momentum).add_(var, alpha=momentum * (n / (n - 1) if n > 1 else 1.0))
            sc, sh = ops.abn_fold(mean, var, weight, bias, eps)
            st = torch.stack([mean, var, sc, sh])
        elif training:
            st = ops.abn_stats(x, weight, bias, eps, momentum, running_mean, running_var)
        else:
            sc, sh = ops.abn_fold(running_mean, running_var, weight, bias, eps)
            st = torch.stack([running_mean, running_var, sc, sh])
        out = ops.abn_apply(x, st[2], st[3], activation, slope, residual=residual, chan_mul=chan_mul)
        # without a fused residual the backward recomputes the activation's sign from x (same FMA as the apply pass): the stored
        # output is not read again -- two HBM passes fewer per layer
        ctx.out_saved = residual is not None or activation == "elu"
        ctx.save_for_backward(x, out if ctx.out_saved else None, st, weight, chan_mul)
        ctx.params = (weight, bias)
        ctx.cfg = (training, eps, activation, slope, residual is not None)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        x, out, st, weight, chan_mul = ctx.saved_tensors
        training, eps, activation, slope, has_res = ctx.cfg
        # eval mode (libs/functions.py:144-147): edz = eydz = 0 -> dx = dz * gamma * rsqrt(var + eps), and -- a quirk of the
        # reference kept as is -- dweight = sign(w) * eydz * n = 0, dbias = edz * n = 0
        wparam, bparam = ctx.params
        gw = _direct_grad(wparam) if (training and ctx.needs_input_grad[1]) else None
        gb = _direct_grad(bparam) if (training and ctx.needs_input_grad[2]) else None
        if gw is None or gb is None:
            gw = gb = None
        dx, dres, dw, db = ops.abn_backward(x, out, ops.to_nhwc(dout), st, weight, eps, activation, slope, chan_mul, has_res,
                                            training=training, dweight_out=gw, dbias_out=gb, sync_fn=_sync_mean if ctx.sync else None)
        if gw is not None:                                   # the reduce kernel wrote dweight / dbias into the flat gradient buffer
            _grad_written(wparam); _grad_written(bparam)
            dw = db = None
        return dx, dw, db, None, None, None, None, None, None, None, dres, None, None


# ------------------------------------------------------------------------------------------------ ESPNet-C (networks/espnet.py)
# Activations between ESPNet-C layers are dense NHWC tensors whose channel count is padded to a multiple of 4 (19 -> 20, 25 -> 28,
# 131 -> 132) with zero pad channels, so every convolution reads them in place; weights are zero-padded to match.
def _esp_conv(x, w_ohwi, stride, pad, dil, precise):
    """Forward convolution of a channel-padded input with channel-padded OHWI weights; 3xTF32 when `precise`."""
    if precise:
        return ops.conv2d_fwd_3xtf32(x, w_ohwi, stride, pad, dil)
    return ops.conv2d_fwd(x, w_ohwi, stride, pad, dil)


def _esp_wgrad(x, dy, weight, stride, pad, dil):
    """(Cout, Cin, KH, KW)-shaped weight gradient (a view of the channel-padded OHWI result).  Main stream: autograd accumulates the
    returned view into .grad right away."""
    cout, cin, kh, kw = weight.shape
    dw = ops.conv2d_wgrad(x, dy, (kh, kw), stride, pad, dil)
    return dw[:cout, :, :, :cin].permute(0, 3, 1, 2)


def _esp_weight(weight, cin_p):
    w = ops.weight_ohwi(weight)
    return _padded_weight(w, ops.pad4(w.shape[0]), cin_p)


class EspConv(torch.autograd.Function):
    """One convolution between channel-padded NHWC tensors (ESPNet-C's classifier): (N, pad4(Cout), OH, OW) out, zero pad channels."""

    @staticmethod
    def forward(ctx, x, weight, stride, pad, dil, precise):
        wp = _esp_weight(weight, x.shape[1])
        y = _esp_conv(x, wp, stride, pad, dil, precise)
        ctx.save_for_backward(x, wp, weight)
        ctx.cfg = (stride, pad, dil)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, wp, weight = ctx.saved_tensors
        stride, pad, dil = ctx.cfg
        dy = ops.to_nhwc(dy)
        dx = ops.conv2d_dgrad(dy, wp, tuple(x.shape), stride, pad, dil) if ctx.needs_input_grad[0] else None
        dw = _esp_wgrad(x, dy, weight, stride, pad, dil) if ctx.needs_input_grad[1] else None
        return dx, dw, None, None, None, None


def _bn_stats(x, training, momentum, rm, rv, nbt):
    if training:
        return ops.bnprelu_stats(x, momentum, rm, rv, nbt)
    return torch.stack([rm, rv])


class EspBnPrelu(torch.autograd.Function):
    """BatchNorm2d(eps) + PReLU over the channel concatenation of `pieces` (and, with `image`, its average pooling `ipa_times` times,
    the InputProjectionA channels): ESPNet-C's CBR after its convolution and the BR blocks b1 / b2 / b3.  The concatenation is one
    channel-padded NHWC buffer; the pooled image is written straight into its slice (forward only: the image has no gradient).
    Returns the channel-padded output and, for b1, the pooled image slice that b2's projection pools once more."""

    @staticmethod
    def forward(ctx, image, ipa, weight, bias, alpha, running_mean, running_var, nbt, training, momentum, eps, *pieces):
        n, _, h, w = pieces[0].shape
        widths = [p.shape[1] for p in pieces]
        c = sum(widths) + (3 if image is not None else 0)
        cp = ops.pad4(c)
        if len(pieces) == 1 and image is None and ops.nhwc_meta(pieces[0])[4] == c:
            x = pieces[0]
        else:
            x = ops.empty_nhwc(n, c, h, w, pieces[0].device, pitch=cp)
            off = 0
            for p, k in zip(pieces, widths):
                ops.slice_copy(p, 0, x, off, k)
                off += k
            if image is not None:
                src = image
                for _ in range(ipa):
                    hh, ww = (src.shape[2] + 1) // 2, (src.shape[3] + 1) // 2
                    dst = x[:, off:off + 3] if (hh, ww) == (h, w) else ops.empty_nhwc(n, 3, hh, ww, x.device)
                    ops.avgpool3x3s2(src, dst)
                    src = dst
        st = _bn_stats(x, training, momentum, running_mean, running_var, nbt)
        y = ops.bnprelu_apply(x, st[0], st[1], weight, bias, alpha, eps, out_channels=cp)
        ctx.save_for_backward(x, st, weight, bias, alpha)
        ctx.cfg = (training, eps, widths)
        projected = x[:, c - 3:c] if image is not None else None
        if projected is not None:
            ctx.mark_non_differentiable(projected)
        return y, projected

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, _dproj):
        x, st, weight, bias, alpha = ctx.saved_tensors
        training, eps, widths = ctx.cfg
        dy = ops.to_nhwc(dy)
        dw, db, da, coef = ops.bnprelu_bwd_reduce(x, dy, st[0], st[1], weight, bias, alpha, eps)
        dx = ops.bnprelu_bwd_dx(x, dy, st[0], st[1], weight, bias, alpha, eps, training, coef, dx_channels=ops.pad4(x.shape[1]))
        dpieces, off = [], 0
        if len(widths) == 1 and dx.shape[1] == widths[0]:
            dpieces = [dx]
        else:
            n, _, h, w = dx.shape
            for k in widths:
                d = ops.empty_nhwc(n, k, h, w, dx.device)
                ops.slice_copy(dx, off, d, 0, k)
                dpieces.append(d)
                off += k
        return (None, None, dw, db, da, None, None, None, None, None, None) + tuple(dpieces)


class EspBlock(torch.autograd.Function):
    """One ESP module of ESPNet-C -- DownSamplerB (`c1` 3x3 / stride 2) or DilatedParllelResidualBlockB (`c1` 1x1, residual `add`):
    reduce -> five dilated 3x3 branches (d = 1, 2, 4, 8, 16) -> hierarchical feature fusion + concatenation (+ input) -> BatchNorm ->
    PReLU.  Forward: six wgmma convolutions (3xTF32 when `precise`), then one pass that forms the combine and its batch statistics,
    then the BN + PReLU apply.  Backward: one reduce pass and one pass that writes every branch's gradient (suffix sums of the fused
    slices) and the residual's; the five branch data gradients are summed into d(c1 out) through the convolution epilogue's residual
    input, in a fixed order."""

    @staticmethod
    def forward(ctx, x, w_c1, w_d1, w_d2, w_d4, w_d8, w_d16, bn_w, bn_b, alpha, running_mean, running_var, nbt, stride, add, training,
                momentum, eps, precise):
        n_red, n1 = w_d2.shape[0], w_d1.shape[0]
        k = w_c1.shape[2]
        wc1 = _esp_weight(w_c1, x.shape[1])
        t = _esp_conv(x, wc1, stride, (k - 1) // 2, 1, precise)                         # (N, pad4(n), H', W')
        wbr = [_esp_weight(wd, t.shape[1]) for wd in (w_d1, w_d2, w_d4, w_d8, w_d16)]
        outs = [_esp_conv(t, wb, 1, d, d, precise) for wb, d in zip(wbr, (1, 2, 4, 8, 16))]
        branches = [outs[0][:, :n1]] + [o[:, :n_red] for o in outs[1:]]
        N, _, h, w = t.shape
        c = n1 + 4 * n_red
        comb = ops.empty_nhwc(N, c, h, w, x.device)
        if training:
            st = ops.esp_combine(branches, x if add else None, comb, momentum, running_mean, running_var, nbt)
        else:
            ops.esp_combine(branches, x if add else None, comb, stats=False)
            st = torch.stack([running_mean, running_var])
        y = ops.bnprelu_apply(comb, st[0], st[1], bn_w, bn_b, alpha, eps, out_channels=ops.pad4(c))
        ctx.save_for_backward(x, t, comb, st, wc1, *wbr, w_c1, w_d1, w_d2, w_d4, w_d8, w_d16, bn_w, bn_b, alpha)
        ctx.cfg = (stride, add, training, eps, n1, n_red)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, t, comb, st, wc1, *rest = ctx.saved_tensors
        wbr, params = rest[:5], rest[5:]
        w_c1, w_d1, w_d2, w_d4, w_d8, w_d16, bn_w, bn_b, alpha = params
        stride, add, training, eps, n1, n_red = ctx.cfg
        dy = ops.to_nhwc(dy)
        dbw, dbb, da, coef = ops.bnprelu_bwd_reduce(comb, dy, st[0], st[1], bn_w, bn_b, alpha, eps)
        dds, dres = ops.esp_bwd_dx(comb, dy, st[0], st[1], bn_w, bn_b, alpha, eps, training, coef, n1, n_red,
                                   add and ctx.needs_input_grad[0])
        dt = None
        for dd, wb, d in zip(dds, wbr, (1, 2, 4, 8, 16)):                # d(c1 out) = sum of the branch data gradients, in order
            dt = ops.conv2d_dgrad(dd, wb, tuple(t.shape), 1, d, d, residual=dt)
        k = w_c1.shape[2]
        dx = None
        if ctx.needs_input_grad[0]:
            if stride == 1:
                dx = ops.conv2d_dgrad(dt, wc1, tuple(x.shape), 1, (k - 1) // 2, 1, residual=dres)
            else:
                dx = ops.conv2d_dgrad(dt, wc1, tuple(x.shape), stride, (k - 1) // 2, 1)
                assert dres is None
        dws = [_esp_wgrad(t, dd, wd, 1, d, d) for dd, wd, d in zip(dds, (w_d1, w_d2, w_d4, w_d8, w_d16), (1, 2, 4, 8, 16))]
        dwc1 = _esp_wgrad(x, dt, w_c1, stride, (k - 1) // 2, 1)
        return (dx, dwc1, *dws, dbw, dbb, da) + (None,) * 9


class EspConvTranspose(torch.autograd.Function):
    """nn.ConvTranspose2d(Cin, Cout, 2, stride=2, bias=False) between channel-padded NHWC tensors (the full ESPNet's up_l3, up_l2 and
    classifier): (N, pad4(Cout), 2h, 2w) out, zero pad channels.  `weight` is the (Cin, Cout, 2, 2) parameter.
      forward: per output-row parity a, one 1x1 GEMM to 2 * pad4(Cout) channels (the two output columns), 3xTF32, written onto the
               every-other-row sub-grid (ops.conv_transpose2x2_fwd);
      dgrad:   dx = conv2d(dy, w[ci][a][b][co], 2x2, stride 2) -- a forward wgmma convolution;
      wgrad:   the weight gradient of that same convolution, with dy as its input and x as its output gradient."""

    @staticmethod
    def forward(ctx, x, weight):
        cin, cout = weight.shape[:2]
        cin_p, cout_p = x.shape[1], ops.pad4(cout)
        wr = torch.zeros((2, 2, cout_p, cin_p), device=weight.device, dtype=torch.float32)
        wr[:, :, :cout, :cin] = weight.permute(2, 3, 1, 0)               # [a][b][co][ci]
        y = ops.conv_transpose2x2_fwd(x, wr.reshape(2, 2 * cout_p, 1, 1, cin_p))
        ctx.save_for_backward(x, weight)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        cin, cout = weight.shape[:2]
        cin_p = x.shape[1]
        dy = ops.to_nhwc(dy)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            wd = torch.zeros((cin_p, 2, 2, dy.shape[1]), device=weight.device, dtype=torch.float32)
            wd[:cin, :, :, :cout] = weight.permute(0, 2, 3, 1)            # [ci][a][b][co]: OHWI of the 2x2 / stride-2 convolution of dy
            dx = ops.conv2d_fwd(dy, wd, 2, 0, 1)
        if ctx.needs_input_grad[1]:
            dw = ops.conv2d_wgrad(dy, x, (2, 2), 2, 0, 1)[:cin, :, :, :cout].permute(0, 3, 1, 2)
        return dx, dw


class EspConcat(torch.autograd.Function):
    """torch.cat(pieces, 1) into one channel-padded NHWC buffer (zero pad channels) for the convolution that reads it."""

    @staticmethod
    def forward(ctx, *pieces):
        n, _, h, w = pieces[0].shape
        widths = [p.shape[1] for p in pieces]
        c = sum(widths)
        x = torch.zeros((n, h, w, ops.pad4(c)), device=pieces[0].device, dtype=torch.float32).permute(0, 3, 1, 2)
        off = 0
        for p, k in zip(pieces, widths):
            ops.slice_copy(p, 0, x, off, k)
            off += k
        ctx.widths = widths
        return x

    @staticmethod
    @once_differentiable
    def backward(ctx, dx):
        dx = ops.to_nhwc(dx)
        n, _, h, w = dx.shape
        out, off = [], 0
        for k in ctx.widths:
            d = ops.empty_nhwc(n, k, h, w, dx.device)
            ops.slice_copy(dx, off, d, 0, k)
            out.append(d)
            off += k
        return tuple(out)


# ------------------------------------------------------------------------------------------------ MobileNetV2 (networks/mobilenet.py)
# Activations are dense NHWC tensors (every MobileNetV2 width is a multiple of 8).  The 1x1 expand / project convolutions and the stem
# are Conv2d above; these two Functions are the rest of an inverted residual.  Saved for backward: each BatchNorm's input (z is
# recomputed from it for the ReLU6 mask, never stored) and each convolution's input, i.e. the activated expansion is stored, not
# recomputed (DESIGN.md "MobileNetV2 student" has the memory this takes).
class MbBnAct(torch.autograd.Function):
    """nn.BatchNorm2d followed by nn.ReLU6 (`relu6`: the stem and the 1x1 expansions), or the linear BatchNorm of an inverted
    residual's projection plus, when the block has one, its input (`residual`: x + bn(conv(x)))."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, nbt, training, momentum, eps, relu6, residual):
        st = _bn_stats(x, training, momentum, running_mean, running_var, nbt)
        y = ops.bnact_apply(x, st[0], st[1], weight, bias, eps, relu6, residual)
        ctx.save_for_backward(x, st, weight, bias)
        ctx.cfg = (training, eps, relu6, residual is not None)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, st, weight, bias = ctx.saved_tensors
        training, eps, relu6, has_res = ctx.cfg
        dy = ops.dense_nhwc(dy)
        dw, db, coef = ops.bnact_bwd_reduce(x, dy, st[0], st[1], weight, bias, eps, relu6)
        dx = ops.bnact_bwd_dx(x, dy, st[0], st[1], weight, bias, eps, relu6, training, coef)
        dres = dy if has_res and ctx.needs_input_grad[10] else None
        return dx, dw, db, None, None, None, None, None, None, None, dres


class MbDwBnRelu6(torch.autograd.Function):
    """Depthwise 3x3 convolution (stride 1 or 2, padding = dilation) -> BatchNorm2d -> ReLU6 of an inverted residual.  In training
    the convolution's pass also forms the BatchNorm's batch statistics, so its output is not read a second time for them."""

    @staticmethod
    def forward(ctx, x, w_dw, weight, bias, running_mean, running_var, nbt, stride, dilation, training, momentum, eps):
        x = ops.dense_nhwc(x)
        t, st = ops.dwconv3x3_fwd(x, w_dw, stride, dilation, training, momentum, running_mean, running_var, nbt)
        if not training:
            st = torch.stack([running_mean, running_var])
        y = ops.bnact_apply(t, st[0], st[1], weight, bias, eps, True)
        ctx.save_for_backward(x, t, st, w_dw, weight, bias)
        ctx.cfg = (stride, dilation, training, eps)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, t, st, w_dw, weight, bias = ctx.saved_tensors
        stride, dilation, training, eps = ctx.cfg
        dy = ops.dense_nhwc(dy)
        dbw, dbb, coef = ops.bnact_bwd_reduce(t, dy, st[0], st[1], weight, bias, eps, True)
        dt = ops.bnact_bwd_dx(t, dy, st[0], st[1], weight, bias, eps, True, training, coef)
        dx = ops.dwconv3x3_dgrad(dt, w_dw, tuple(x.shape), stride, dilation) if ctx.needs_input_grad[0] else None
        dwd = ops.dwconv3x3_wgrad(x, dt, stride, dilation) if ctx.needs_input_grad[1] else None
        return (dx, dwd, dbw, dbb) + (None,) * 8


class ResampleBilinear(torch.autograd.Function):
    """F.interpolate(t, (H, W), mode='bilinear', align_corners=True) with a gradient: the forward is the teacher resample kernel, the
    backward its adjoint as a fixed-order gather (no float atomics, so two runs of a step stay bit-identical).  The full ESPNet's
    logits reach the discriminator this way, resized onto the teacher's logit grid."""

    @staticmethod
    def forward(ctx, t, H, W):
        ctx.hw = tuple(t.shape[2:])
        return ops.resample_nhwc(t, H, W)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return ops.resample_adjoint_nhwc(g, *ctx.hw), None, None


class MaxPool3x3s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y, arg = ops.maxpool_fwd(x)
        ctx.save_for_backward(arg)
        ctx.shape = x.shape
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        (arg,) = ctx.saved_tensors
        return ops.maxpool_bwd(ops.to_nhwc(dy), arg, ctx.shape)


class PspPool(torch.autograd.Function):
    """AdaptiveAvgPool2d(1/2/3/6) of the PSP module in one launch -> (N, 50, C)."""

    @staticmethod
    def forward(ctx, x, sizes):
        ctx.sizes, ctx.shape = sizes, x.shape
        return ops.psp_pool_fwd(x, list(sizes))

    @staticmethod
    @once_differentiable
    def backward(ctx, dp):
        return ops.psp_pool_bwd(dp.contiguous(), list(ctx.sizes), ctx.shape), None


class PspAssemble(torch.autograd.Function):
    """torch.cat([upsample(stage_i)..., feats], 1) written in place into one NHWC buffer (pspnet_combine.py:110-111)."""

    @staticmethod
    def forward(ctx, feats, sizes, *stages):
        n, c, h, w = feats.shape
        cs = stages[0].shape[2]
        ctot = len(stages) * cs + c
        buf = ops.empty_nhwc(n, ctot, h, w, feats.device)
        for i, (s, stg) in enumerate(zip(sizes, stages)):
            ops.psp_upsample_fwd(stg.contiguous(), s, buf, i * cs)
        ops.slice_copy(feats, 0, buf, len(stages) * cs, c)
        ctx.cfg = (sizes, cs, c, feats.shape)
        return buf

    @staticmethod
    @once_differentiable
    def backward(ctx, dbuf):
        sizes, cs, c, fshape = ctx.cfg
        dbuf = ops.to_nhwc(dbuf)
        dfe = ops.empty_nhwc(fshape[0], c, fshape[2], fshape[3], dbuf.device)
        ops.slice_copy(dbuf, len(sizes) * cs, dfe, 0, c)
        dst = tuple(ops.psp_upsample_bwd(dbuf, s, cs, i * cs) for i, s in enumerate(sizes))
        return (dfe, None) + dst
