"""Execution engine of the SAGAN discriminator on the sm_90a kernels (csrc/disc.cu + the wgmma convolutions).

Three passes over the same parameters, none of them through torch operators or autograd:

  forward(x)            networks/sagan_models.py:156-168 (+ spectral.py:23-35 power iteration per SN layer, BN2d batch stats)
  backward(tape, gout)  first-order reverse pass: parameter gradients and, on request, d out / d x
  gp_forward / gp_backward   CriterionAdditionalGP (utils/criterion.py:98-120) WITHOUT double backward: the first-order chain to
                        the input gives g = d(sum D(x))/dx and the penalty value; the parameter gradient is "reverse over
                        forward" -- a tangent pass along v = c_n g_n, then one reverse pass over the joint (primal, tangent)
                        graph, which for the bilinear layers is the ordinary backward over a [primal | tangent] batch of 2B.
                        oracle/gp_dual.py states the same operation sequence in torch and is pinned against autograd.

Activations are NHWC rows.  The 4x4/s2 spectral-norm convolutions and the q/k/v projections run on the wgmma implicit-GEMM
kernel in split precision (3xTF32); weight gradients on the wgmma wgrad kernel (TF32); 1/sigma rides in the convolution
epilogue's per-channel scale, so no normalised weight tensor is ever materialised.
"""
import ctypes

import torch

from .. import ops
from .._cabi import lib

LEAK = 0.1
ACT_NONE, ACT_LEAKY = 0, 1


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _f(*shape, dev):
    return torch.empty(shape, device=dev, dtype=torch.float32)


class _Tape:
    pass


class _SnLayer(ctypes.Structure):
    """struct skd_sn_layer (include/skd.h)"""
    _fields_ = [("Cout", ctypes.c_int), ("taps", ctypes.c_int), ("Cin", ctypes.c_int), ("vec_len", ctypes.c_int),
                ("w_bar", ctypes.c_void_p), ("u", ctypes.c_void_p), ("v", ctypes.c_void_p), ("u_save", ctypes.c_void_p),
                ("v_save", ctypes.c_void_p), ("sigma", ctypes.c_void_p), ("inv_sigma_vec", ctypes.c_void_p)]


class DiscEngine:
    """Bound to one `Discriminator` module; reads its parameters in place (FlatSGD views included)."""

    def __init__(self, D):
        self.D = D
        self.precise = True            # split-precision (3xTF32) forward / data-gradient convolutions
        self.split_k = True            # split-K for the convolutions with too few output tiles to fill the GPU
        self._prep = None
        self._ws = None

    # ------------------------------------------------------------------------------------------------ static description
    def _sn_layers(self):
        D = self.D
        return [l[0].module for l in (D.l1, D.l2, D.l3, D.l4)[:D.n_sn_layers]]

    def _attn_after(self, li):
        """attention module that follows SN layer index li (sagan_models.py:160-165), or None"""
        D = self.D
        if li == 2:
            return D.attn1
        if li == 3:
            return D.attn2
        return None

    def _workspaces(self, dev):
        if self._ws is None or self._ws["dev"] != dev:
            L = lib()
            self._ws = dict(dev=dev,
                            bn=torch.zeros(L.skd_bn2d_workspace_doubles(), device=dev, dtype=torch.float64),
                            sn=torch.zeros(L.skd_sn_weight_grad_workspace_doubles(), device=dev, dtype=torch.float64))
        return self._ws

    # ------------------------------------------------------------------------------------------------ per-step weight staging
    def prepare(self):
        """Pin one staging of the weights for several passes (NetModel: once per discriminator phase, the parameters being
        constant within it); release() un-pins.  An un-pinned forward() stages on every call."""
        self._prep = self._stage()
        return self._prep

    def _stage(self):
        """Channel-padded / lo-part / data-gradient / transposed copies of the weights."""
        L, st = lib(), _st()
        D = self.D
        dev = D.last[0].weight.device
        prep = dict(layers=[], attn={})
        for m in self._sn_layers():
            w = m.weight_bar                                     # (Cout, Cin, 4, 4) in channels-last (OHWI) storage
            cout, cin = w.shape[0], w.shape[1]
            if w.stride() != (16 * cin, 1, 4 * cin, cin):
                raise ValueError("Non-contiguous input")          # weight_bar must be OHWI-stored
            cin_p = ops.pad4(cin)
            w_hi, w_lo = _f(cout, 16, cin_p, dev=dev), _f(cout, 16, cin_p, dev=dev)
            L.skd_disc_weight_prep(cout * 16, cin, cin_p, _p(w), _p(w_hi), _p(w_lo), st)
            wd, wd_lo = _f(4 * cin_p, 9, cout, dev=dev), _f(4 * cin_p, 9, cout, dev=dev)
            L.skd_disc_dgrad_weight_prep(cout, cin, cin_p, _p(w), _p(wd), _p(wd_lo), st)
            prep["layers"].append(dict(m=m, cin=cin, cin_p=cin_p, cout=cout, w_hi=w_hi, w_lo=w_lo, wd=wd, wd_lo=wd_lo))
        for key, A in (("attn1", D.attn1), ("attn2", D.attn2)):
            if A is None:
                continue
            c, d = A.chanel_in, A.query_conv.out_channels
            ldq = 2 * d + c
            w, w_lo = _f(ldq, c, dev=dev), _f(ldq, c, dev=dev)
            off = 0
            for conv in (A.query_conv, A.key_conv, A.value_conv):
                rows = conv.out_channels
                L.skd_disc_weight_prep(rows, c, c, _p(conv.weight), _p(w[off:]), _p(w_lo[off:]), st)
                off += rows
            wt, wt_lo = _f(c, ldq, dev=dev), _f(c, ldq, dev=dev)
            L.skd_weight_flip_transpose(ldq, c, 1, 1, _p(w), _p(wt), 0, st)
            L.skd_split_tf32(wt.numel(), _p(wt), None, _p(wt_lo), st)
            bias = torch.cat([A.query_conv.bias, A.key_conv.bias, A.value_conv.bias]).detach()
            prep["attn"][key] = dict(A=A, c=c, d=d, ldq=ldq, w=w, w_lo=w_lo, wt=wt, wt_lo=wt_lo, bias=bias)
        return prep

    def release(self):
        self._prep = None

    # ------------------------------------------------------------------------------------------------ helpers
    def _conv(self, n, h, w, cin, cout, k, stride, pad, x, x_lo, ldx, wgt, wgt_lo, y, ldy, out_hw=(0, 0), scale=None, shift=None,
              residual=None, ldr=0, act=ACT_NONE, slope=0.0):
        if not self.precise:
            x_lo = wgt_lo = None
        L = lib()
        # few output tiles + long K (4x8 .. 16x32 maps): split-K over (tile, K range) units, partial planes in a workspace
        nws = L.skd_conv2d_fwd_sm100_splitk_workspace_floats(n, h, w, cin, cout, k, k, stride, pad, 1, out_hw[0], out_hw[1]) if self.split_k else 0
        ws = torch.empty(nws, device=y.device, dtype=torch.float32) if nws else None
        L.skd_conv2d_fwd_sm100_splitk(n, h, w, cin, cout, k, k, stride, pad, 1, _p(x), _p(x_lo), ldx, _p(wgt), _p(wgt_lo), _p(y), ldy,
                                      out_hw[0], out_hw[1], _p(scale), _p(shift), _p(residual), ldr, act, slope, _p(ws), nws, _st())

    def _split(self, t, rows=None):
        """lo part of the first `rows` leading entries of t (whole tensor by default), same shape as t"""
        lo = torch.empty_like(t)
        if self.precise:
            n = t.numel() if rows is None else rows * (t.numel() // t.shape[0])
            lib().skd_split_tf32(n, _p(t), None, _p(lo), _st())
        return lo

    @staticmethod
    def _half(t, B, second):
        return t[B:] if second else t[:B]

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self, x, room_for_tangent=False, need_out=True):
        """x: (B, C, H, W) with any (image, channel, pixel) strides.  Returns the tape; tape.out is (B, 1, OH, OW)."""
        ops._f32(x)
        L, st = lib(), _st()
        D = self.D
        prep = self._prep if self._prep is not None else self._stage()
        dev = x.device
        ws = self._workspaces(dev)
        B, C, H, W = x.shape
        cap = 2 * B if room_for_tangent else B
        t = _Tape()
        t.B, t.cap, t.x, t.xs, t.C, t.H, t.W = B, cap, x, ops.pixel_strides(x), C, H, W
        t.prep = prep
        # ---- spectral norm: one power iteration per layer; u, v advance in place (spectral.py:28-31)
        t.sn = []
        descs = (_SnLayer * len(prep["layers"]))()
        for i, lay in enumerate(prep["layers"]):
            m = lay["m"]
            vec = max(lay["cout"], 4 * lay["cin_p"])
            s = dict(u=_f(lay["cout"], dev=dev), v=_f(16 * lay["cin"], dev=dev), sigma=_f(1, dev=dev), inv=_f(vec, dev=dev))
            descs[i] = _SnLayer(lay["cout"], 16, lay["cin"], vec, _p(m.weight_bar), _p(m.weight_u), _p(m.weight_v), _p(s["u"]), _p(s["v"]),
                                _p(s["sigma"]), _p(s["inv"]))
            t.sn.append(s)
        # all four layers in one call: each phase of the iteration is a grid over every layer (csrc/disc.cu, sn_phase*_kernel)
        sn_ws = _f(L.skd_sn_power_iter_batched_workspace_floats(len(descs), ctypes.cast(descs, ctypes.c_void_p)), dev=dev)
        L.skd_sn_power_iter_batched(len(descs), ctypes.cast(descs, ctypes.c_void_p), _p(sn_ws), st)
        # ---- preprocess (sagan_models.py:147,157): BatchNorm2d with batch statistics in train mode
        bn = D.preprocess_additional
        Cp = ops.pad4(C)
        t.Cp = Cp
        t.h0, t.h0_lo = _f(cap, H, W, Cp, dev=dev), _f(cap, H, W, Cp, dev=dev)
        if D.preprocess_mode == 1:
            t.mean, t.rstd = _f(32, dev=dev), _f(32, dev=dev)
            if bn.training:
                L.skd_bn2d_stats(B, C, H * W, _p(x), *t.xs, bn.eps, bn.momentum, _p(bn.running_mean), _p(bn.running_var),
                                 _p(bn.num_batches_tracked), _p(t.mean), _p(t.rstd), _p(ws["bn"]), st)
            else:
                t.mean[:C] = bn.running_mean
                t.rstd[:C] = torch.rsqrt(bn.running_var + bn.eps)
            L.skd_bn2d_apply(B, C, H * W, _p(x), *t.xs, _p(t.mean), _p(t.rstd), _p(bn.weight), _p(bn.bias), _p(t.h0),
                             _p(t.h0_lo) if self.precise else None, Cp, st)
        else:
            raise NotImplementedError("preprocess_GAN_mode 2 / 3 (tanh / rescale) are not on the distillation path (run_train_val.sh uses 1)")
        # ---- SN conv -> LeakyReLU(0.1) stacks, attention after l3 and l4 (sagan_models.py:158-165)
        t.h, t.h_lo, t.dims, t.att = [], [], [(H, W)], {}
        hin, hin_lo, hc, wc = t.h0, t.h0_lo, H, W
        for li, (lay, s) in enumerate(zip(prep["layers"], t.sn)):
            oh, ow = (hc + 2 - 4) // 2 + 1, (wc + 2 - 4) // 2 + 1
            if oh < 1 or ow < 1:
                raise ValueError("input map too small for the discriminator")
            cout = lay["cout"]
            h = _f(cap, oh, ow, cout, dev=dev)
            self._conv(B, hc, wc, lay["cin_p"], cout, 4, 2, 1, hin, hin_lo, lay["cin_p"], lay["w_hi"], lay["w_lo"], h, cout,
                       scale=s["inv"], shift=lay["m"].bias, act=ACT_LEAKY, slope=LEAK)
            h_lo = self._split(h, B)
            t.h.append(h); t.h_lo.append(h_lo); t.dims.append((oh, ow))
            hin, hin_lo, hc, wc = h, h_lo, oh, ow
            A = self._attn_after(li)
            if A is not None:
                a = prep["attn"]["attn1" if li == 2 else "attn2"]
                n = oh * ow
                qkv = _f(cap * n, a["ldq"], dev=dev)
                self._conv(1, 1, B * n, a["c"], a["ldq"], 1, 1, 0, h, h_lo, a["c"], a["w"], a["w_lo"], qkv, a["ldq"], shift=a["bias"])
                attn, o = _f(cap, n, n, dev=dev), _f(cap * n, a["c"], dev=dev)
                y, y_lo = _f(cap, oh, ow, a["c"], dev=dev), _f(cap, oh, ow, a["c"], dev=dev)
                L.skd_attn_fwd(B, n, a["c"], a["d"], _p(qkv), a["ldq"], _p(h), _p(A.gamma), _p(attn), _p(o), _p(y),
                               _p(y_lo) if self.precise else None, st)
                t.att[li] = dict(a=a, n=n, qkv=qkv, attn=attn, o=o, y=y, y_lo=y_lo)
                hin, hin_lo = y, y_lo
        t.top, t.top_lo, t.top_hw = hin, hin_lo, (hc, wc)
        # ---- last conv (sagan_models.py:140,166).  Size-aware: a map smaller than 4x4 uses the top-left window of the kernel
        last = D.last[0]
        t.kh, t.kw = min(4, hc), min(4, wc)
        t.ohw = (hc - t.kh + 1, wc - t.kw + 1)
        t.ctop = last.weight.shape[1]
        if need_out:
            t.out = _f(B, 1, t.ohw[0], t.ohw[1], dev=dev)
            L.skd_disc_last_fwd(B, hc, wc, t.ctop, t.kh, t.kw, _p(hin), _p(last.weight), 4 * t.ctop, _p(last.bias), _p(t.out), st)
        return t

    # ------------------------------------------------------------------------------------------------ reverse pass
    def _grad_buf(self, sink, name, param):
        """-> (tensor to write, accumulate flag).  sink: dict name -> fresh gradient, or None = accumulate into param.grad."""
        if sink is None:
            return param.grad, 1
        if name in sink:
            return sink[name], 1
        g = torch.empty_like(param)
        sink[name] = g
        return g, 0

    def _reverse_layers(self, t, g_top, joint, sink, param_grads, need_input_adj):
        """Reverse pass through the conv / attention stack from the adjoint of the last conv's input.  joint: rows are
        [primal | tangent] (2B images); masks and attention maps come from the primal half.  Returns the adjoint of the
        BatchNorm output [nb][H][W][Cp] (None when not needed)."""
        L, st = lib(), _st()
        D = self.D
        dev = g_top.device
        B = t.B
        nb = 2 * B if joint else B
        ws = self._workspaces(dev)
        names = D.sn_names
        g = g_top                                                     # adjoint of the current layer's OUTPUT, [nb][oh][ow][c]
        masked = False                                                 # g already multiplied by the layer's LeakyReLU mask
        for li in range(len(t.prep["layers"]) - 1, -1, -1):
            lay, s = t.prep["layers"][li], t.sn[li]
            oh, ow = t.dims[li + 1]
            hin_hw = t.dims[li]
            cout, cin, cin_p = lay["cout"], lay["cin"], lay["cin_p"]
            if li in t.att:
                # ---- attention: y = gamma O + h  ->  adjoint of h = gqkv Wqkv + gy
                at = t.att[li]; a = at["a"]; n = at["n"]; A = a["A"]
                gqkv = _f(nb * n, a["ldq"], dev=dev)
                wsf = _f(L.skd_attn_bwd_workspace_floats(B, n, a["c"]), dev=dev)
                pre = "attn1." if li == 2 else "attn2."
                gg, acc = self._grad_buf(sink, pre + "gamma", A.gamma) if param_grads else (None, 0)
                g2 = g.view(nb * n, a["c"])
                if joint:
                    gy = None if at.get("primal_adj_zero") else g2[:B * n]
                    L.skd_attn_bwd(B, n, a["c"], a["d"], _p(at["qkv"]), a["ldq"], _p(at["attn"]), _p(at["o"]), _p(A.gamma), _p(gy),
                                   _p(at["qkv"][B * n:]), _p(at["dattn"]), _p(at["o"][B * n:]), _p(g2[B * n:]), _p(gqkv), _p(gqkv[B * n:]),
                                   _p(gg), acc, _p(wsf), st)
                else:
                    L.skd_attn_bwd(B, n, a["c"], a["d"], _p(at["qkv"]), a["ldq"], _p(at["attn"]), _p(at["o"]), _p(A.gamma), _p(g2),
                                   None, None, None, None, _p(gqkv), None, _p(gg), acc, _p(wsf), st)
                hx = t.h[li].view(-1, a["c"])                           # attention input rows [cap*n][C]
                if param_grads:
                    dw = _f(a["ldq"], a["c"], dev=dev)
                    nws = L.skd_conv2d_wgrad_sm100_workspace_floats(nb, oh, ow, a["c"], a["ldq"], 1, 1, 1, 0, 1)
                    wsg = _f(max(nws, 4), dev=dev)
                    L.skd_conv2d_wgrad_sm100(nb, oh, ow, a["c"], a["ldq"], 1, 1, 1, 0, 1, _p(hx), a["c"], _p(gqkv), a["ldq"], _p(dw), _p(wsg), st)
                    db = _f(a["ldq"], dev=dev)
                    L.skd_colsum(B * n, a["ldq"], _p(gqkv), a["ldq"], _p(db), st)    # the tangent projections carry no bias
                    off = 0
                    for cname, conv in (("query_conv", A.query_conv), ("key_conv", A.key_conv), ("value_conv", A.value_conv)):
                        r = conv.out_channels
                        self._emit(sink, pre + cname + ".weight", conv.weight, dw[off:off + r].view(r, a["c"], 1, 1))
                        self._emit(sink, pre + cname + ".bias", conv.bias, db[off:off + r])
                        off += r
                gh = _f(nb, oh, ow, a["c"], dev=dev)
                gq_lo = self._split(gqkv)
                self._conv(1, 1, nb * n, a["ldq"], a["c"], 1, 1, 0, gqkv, gq_lo, a["ldq"], a["wt"], a["wt_lo"], gh, a["c"], residual=g2, ldr=a["c"])
                if getattr(t, "debug", None) is not None:
                    t.debug.append(("gy%d" % li, g2.clone())); t.debug.append(("gqkv%d" % li, gqkv.clone())); t.debug.append(("gh%d" % li, gh.clone()))
                g, masked = gh, False
            if not masked:
                gz = torch.empty_like(g)
                per = B * oh * ow * cout
                L.skd_disc_mask_mul(g.numel(), per, _p(t.h[li]), _p(g), _p(gz), None, LEAK, st)
                g = gz
            if getattr(t, "debug", None) is not None:
                t.debug.append(("gz%d" % li, g.clone()))
            # ---- SN conv: z = conv(hin, w_bar) / sigma + b
            hin = t.h0 if li == 0 else (t.att[li - 1]["y"] if (li - 1) in t.att else t.h[li - 1])
            if param_grads:
                m = lay["m"]
                db, acc = self._grad_buf(sink, names[li] + ".bias", m.bias)
                if acc:
                    L.skd_colsum_acc(B * oh * ow, cout, _p(g), cout, _p(db), st)
                else:
                    L.skd_colsum(B * oh * ow, cout, _p(g), cout, _p(db), st)
                dwn = _f(cout, 16, cin_p, dev=dev)
                nws = L.skd_conv2d_wgrad_sm100_workspace_floats(nb, hin_hw[0], hin_hw[1], cin_p, cout, 4, 4, 2, 1, 1)
                wsg = _f(max(nws, 4), dev=dev)
                L.skd_conv2d_wgrad_sm100(nb, hin_hw[0], hin_hw[1], cin_p, cout, 4, 4, 2, 1, 1, _p(hin), cin_p, _p(g), cout, _p(dwn), _p(wsg), st)
                dw, acc = self._grad_buf(sink, names[li] + ".weight_bar", m.weight_bar)
                # d sigma / d w_bar = u v^T with the module's CURRENT u, v, not this forward's: the reference rebinds `u.data` / `v.data`
                # in every forward (spectral.py:30-31) and autograd's saved references to u and v see the latest values, so the backward
                # of D(T) uses the vectors left by the last forward of the phase (D(S), or the penalty's D(interpolated)).  sigma itself
                # is the value this forward computed.  (Visible at batch 1: the rank-one term is as large as the rest of l4's gradient.)
                L.skd_sn_weight_grad(cout, 16, cin, cin_p, _p(dwn), _p(m.weight_bar), _p(m.weight_u), _p(m.weight_v), _p(s["sigma"]), _p(dw), acc,
                                     _p(ws["sn"]), st)
            if li == 0 and not need_input_adj:
                return None
            # data gradient: one 3x3 conv of gz producing the four parity classes, then un-shuffle (+ mask of the layer below)
            hj, wj = (hin_hw[0] + 1) // 2, (hin_hw[1] + 1) // 2
            g_lo = self._split(g)
            d2s = _f(nb, hj, wj, 4 * cin_p, dev=dev)
            self._conv(nb, oh, ow, cout, 4 * cin_p, 3, 1, 1, g, g_lo, cout, lay["wd"], lay["wd_lo"], d2s, 4 * cin_p, out_hw=(hj, wj), scale=s["inv"])
            below_is_leaky = li > 0 and (li - 1) not in t.att
            cq = cin_p if li == 0 else cin
            gprev = _f(nb, hin_hw[0], hin_hw[1], cq, dev=dev)
            L.skd_disc_dgrad_unshuffle(nb, hin_hw[0], hin_hw[1], cin, cin_p, _p(d2s), _p(t.h[li - 1]) if below_is_leaky else None, B, LEAK,
                                       _p(gprev), cq, None, st)
            g, masked = gprev, below_is_leaky
        return g

    def _reverse_bn(self, t, g, joint, sink, param_grads, want_dx, sums_v=None, vdir=None, dense=False):
        """BatchNorm2d(batch statistics) part of the reverse pass: gamma / beta gradients and, on request, d / d x -- in x's own
        layout, or densely as [B][H][W][Cp] (the layout of the penalty's tangent direction)."""
        L, st = lib(), _st()
        D = self.D
        dev = g.device
        B = t.B
        ws = self._workspaces(dev)
        bn = D.preprocess_additional
        C, H, W, Cp = t.C, t.H, t.W, t.Cp
        sums_g = _f(96, dev=dev)
        L.skd_bn2d_reduce(B, C, H * W, _p(t.x), *t.xs, _p(t.mean), _p(t.rstd), _p(g), None, Cp, _p(sums_g), _p(ws["bn"]), st)
        if param_grads:
            sums_t = None
            if joint:
                sums_t = _f(96, dev=dev)
                L.skd_bn2d_reduce(B, C, H * W, _p(t.x), *t.xs, _p(t.mean), _p(t.rstd), _p(g[B:]), _p(vdir), Cp, _p(sums_t), _p(ws["bn"]), st)
            dgam, acc_g = self._grad_buf(sink, "preprocess_additional.weight", bn.weight)
            dbet, acc_b = self._grad_buf(sink, "preprocess_additional.bias", bn.bias)
            if acc_g != acc_b:
                raise RuntimeError("inconsistent gradient sink")
            L.skd_bn2d_param_grad(C, B * H * W, _p(t.rstd), _p(sums_g), _p(sums_t), _p(sums_v), _p(dgam), _p(dbet), acc_g, st)
        if not want_dx:
            return None
        if dense:
            dx = _f(B, H, W, Cp, dev=dev)
            L.skd_bn2d_jacobian(B, C, H * W, _p(t.x), *t.xs, _p(t.mean), _p(t.rstd), _p(bn.weight), _p(g), Cp, _p(sums_g), _p(dx),
                                H * W * Cp, 1, Cp, Cp, None, st)
            return dx
        dx = torch.empty_strided(t.x.shape, t.x.stride(), device=dev, dtype=torch.float32)
        L.skd_bn2d_jacobian(B, C, H * W, _p(t.x), *t.xs, _p(t.mean), _p(t.rstd), _p(bn.weight), _p(g), Cp, _p(sums_g), _p(dx), *ops.pixel_strides(dx),
                            C, None, st)
        return dx

    def _emit(self, sink, name, param, value):
        buf, acc = self._grad_buf(sink, name, param)
        if acc:
            buf.add_(value)
        else:
            buf.copy_(value)

    def backward(self, t, gout, sink, want_dx, param_grads=True):
        """First-order backward of one forward call.  gout: (B,1,OH,OW) adjoint of tape.out."""
        L, st = lib(), _st()
        D = self.D
        dev = gout.device
        B = t.B
        hc, wc = t.top_hw
        last = D.last[0]
        gout = gout.contiguous()
        g = _f(B, hc, wc, t.ctop, dev=dev)
        L.skd_disc_last_dgrad(B, hc, wc, t.ctop, t.kh, t.kw, _p(gout), _p(last.weight), 4 * t.ctop, _p(g), None, st)
        if param_grads:
            gw, acc = self._grad_buf(sink, "last.0.weight", last.weight)
            gb, acc_b = self._grad_buf(sink, "last.0.bias", last.bias)
            if not acc and (t.kh < 4 or t.kw < 4):
                gw.zero_()
            L.skd_disc_last_wgrad(B, hc, wc, t.ctop, t.kh, t.kw, _p(t.top), _p(gout), _p(gw), 4 * t.ctop, _p(gb), acc, st)
        gh0 = self._reverse_layers(t, g, False, sink, param_grads, need_input_adj=want_dx or param_grads)
        if gh0 is None:
            return None
        return self._reverse_bn(t, gh0, False, sink, param_grads, want_dx)

    # ------------------------------------------------------------------------------------------------ WGAN-GP
    def gp_forward(self, x, lambda_gp):
        """Penalty value at the interpolated batch x (criterion.py:105-120).  Advances u, v like the reference's D(interpolated)."""
        L, st = lib(), _st()
        t = self.forward(x, room_for_tangent=True, need_out=False)
        dev = x.device
        B = t.B
        hc, wc = t.top_hw
        last = self.D.last[0]
        g = _f(B, hc, wc, t.ctop, dev=dev)
        L.skd_disc_last_dgrad(B, hc, wc, t.ctop, t.kh, t.kw, None, _p(last.weight), 4 * t.ctop, _p(g), None, st)   # grad_outputs = ones
        # first-order chain to the input, no parameter gradients; BN's input gradient in the dense [B][H][W][Cp] layout
        gh0 = self._reverse_layers(t, g, False, None, False, need_input_adj=True)
        gx = self._reverse_bn(t, gh0, False, None, False, True, dense=True)
        t.g = gx
        t.norms, t.gp = _f(B, dev=dev), torch.empty((), device=dev, dtype=torch.float32)
        L.skd_gp_norms(B, t.H * t.W * t.Cp, _p(gx), float(lambda_gp), _p(t.norms), _p(t.gp), st)
        t.lambda_gp = float(lambda_gp)
        return t

    def gp_backward(self, t, upstream, sink):
        """Parameter gradient of upstream * GP.  upstream: 0-dim device tensor (or None = 1)."""
        L, st = lib(), _st()
        D = self.D
        dev = t.g.device
        B, C, H, W, Cp = t.B, t.C, t.H, t.W, t.Cp
        ws = self._workspaces(dev)
        bn = D.preprocess_additional
        vdir = _f(B, H, W, Cp, dev=dev)
        L.skd_gp_direction(B, H * W * Cp, _p(t.g), _p(t.norms), t.lambda_gp, _p(upstream), _p(vdir), st)
        # ---- tangent forward along v: BN's Jacobian is symmetric -> same kernel as its input gradient
        sums_v = _f(96, dev=dev)
        L.skd_bn2d_reduce(B, C, H * W, _p(t.x), *t.xs, _p(t.mean), _p(t.rstd), _p(vdir), None, Cp, _p(sums_v), _p(ws["bn"]), st)
        L.skd_bn2d_jacobian(B, C, H * W, _p(t.x), *t.xs, _p(t.mean), _p(t.rstd), _p(bn.weight), _p(vdir), Cp, _p(sums_v), _p(t.h0[B:]),
                            H * W * Cp, 1, Cp, Cp, _p(t.h0_lo[B:]) if self.precise else None, st)
        hin, hin_lo, (hc, wc) = t.h0[B:], t.h0_lo[B:], t.dims[0]
        for li, (lay, s) in enumerate(zip(t.prep["layers"], t.sn)):
            oh, ow = t.dims[li + 1]
            cout = lay["cout"]
            tz = _f(B, oh, ow, cout, dev=dev)
            self._conv(B, hc, wc, lay["cin_p"], cout, 4, 2, 1, hin, hin_lo, lay["cin_p"], lay["w_hi"], lay["w_lo"], tz, cout, scale=s["inv"])
            th, th_lo = t.h[li][B:], t.h_lo[li][B:]
            L.skd_disc_mask_mul(tz.numel(), tz.numel(), _p(t.h[li]), _p(tz), _p(th), _p(th_lo) if self.precise else None, LEAK, st)
            hin, hin_lo, hc, wc = th, th_lo, oh, ow
            if li in t.att:
                at = t.att[li]; a = at["a"]; n = at["n"]; A = a["A"]
                tq = at["qkv"][B * n:]
                self._conv(1, 1, B * n, a["c"], a["ldq"], 1, 1, 0, th, th_lo, a["c"], a["w"], a["w_lo"], tq, a["ldq"])     # no bias in the tangent
                at["dattn"] = _f(B, n, n, dev=dev)
                ty, ty_lo = at["y"][B:], at["y_lo"][B:]
                L.skd_attn_tangent_fwd(B, n, a["c"], a["d"], _p(at["qkv"]), _p(tq), a["ldq"], _p(at["attn"]), _p(th), _p(A.gamma),
                                       _p(at["dattn"]), _p(at["o"][B * n:]), _p(ty), _p(ty_lo) if self.precise else None, st)
                hin, hin_lo = ty, ty_lo
        # ---- reverse pass over the joint graph: adjoint of out is 0 (primal) / ones (tangent)
        last = D.last[0]
        g = _f(2 * B, hc, wc, t.ctop, dev=dev)
        g[:B].zero_()
        L.skd_disc_last_dgrad(B, hc, wc, t.ctop, t.kh, t.kw, None, _p(last.weight), 4 * t.ctop, _p(g[B:]), None, st)
        gw, acc = self._grad_buf(sink, "last.0.weight", last.weight)
        if not acc and (t.kh < 4 or t.kw < 4):
            gw.zero_()
        L.skd_disc_last_wgrad(B, hc, wc, t.ctop, t.kh, t.kw, _p(t.top[B:]), None, _p(gw), 4 * t.ctop, None, acc, st)
        gb, acc_b = self._grad_buf(sink, "last.0.bias", last.bias)
        if not acc_b:
            gb.zero_()
        top_li = len(t.prep["layers"]) - 1
        if top_li in t.att:
            t.att[top_li]["primal_adj_zero"] = True
        gh0 = self._reverse_layers(t, g, True, sink, True, need_input_adj=True)
        self._reverse_bn(t, gh0, True, sink, True, False, sums_v=sums_v, vdir=vdir)
        if top_li in t.att:
            t.att[top_li].pop("primal_adj_zero", None)


# ---------------------------------------------------------------------------------------------------- autograd surface
class DiscriminatorFn(torch.autograd.Function):
    """Discriminator.forward as ONE autograd node: [out, p1, p2] (sagan_models.py:168).  The attention maps p1 / p2 are returned
    for inspection only (marked non-differentiable; nothing on the reference's path differentiates through them).
    `params` are listed so that autograd routes their gradients; the engine reads the parameters in place."""

    @staticmethod
    def forward(ctx, D, x, *params):
        t = D.engine.forward(x)
        ctx.D, ctx.tape = D, t
        B = t.B
        maps = []
        for li in (2, 3):
            if li in t.att:
                maps.append(t.att[li]["attn"][:B])
        ctx.mark_non_differentiable(*maps)
        ctx.n_maps = len(maps)
        return (t.out,) + tuple(maps)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout, *unused):
        D, t = ctx.D, ctx.tape
        if t is None:
            raise RuntimeError("Trying to backward through the discriminator a second time")
        want_dx = ctx.needs_input_grad[1]
        want_p = any(ctx.needs_input_grad[2:]) and not D.skip_param_grads
        sink = None if D.accumulate_into_grad else {}
        dx = D.engine.backward(t, gout, sink, want_dx, want_p)
        ctx.tape = None
        ev = getattr(D, "adjoint_done_event", None)
        if ev is not None:                                   # NetModel: the discriminator phase may start on its own stream from here
            ev.record(torch.cuda.current_stream())
        grads = (None,) * (len(ctx.needs_input_grad) - 2)
        if want_p and sink is not None:
            grads = tuple(sink.get(n) for n in D.grad_names)
        return (None, dx) + grads


class GradientPenaltyFn(torch.autograd.Function):
    """CriterionAdditionalGP (utils/criterion.py:98-120) as one node: forward = penalty value (first-order chain to the input),
    backward = its parameter gradient by the tangent + joint reverse pass (no double backward)."""

    @staticmethod
    def forward(ctx, D, x, lambda_gp, *params):
        t = D.engine.gp_forward(x, lambda_gp)
        ctx.D, ctx.tape = D, t
        return t.gp

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        D, t = ctx.D, ctx.tape
        sink = None if D.accumulate_into_grad else {}
        D.engine.gp_backward(t, go.contiguous().float(), sink)
        ctx.tape = None
        grads = (None,) * (len(ctx.needs_input_grad) - 3)
        if sink is not None:
            grads = tuple(sink.get(n) for n in D.grad_names)
        return (None, None, None) + grads


class AdvLossFn(torch.autograd.Function):
    """CriterionAdv / CriterionAdvForG (utils/criterion.py:129-166): value and d loss / d out in one launch.
    kind 0: wgan-gp D loss, 1: hinge D loss, 2: generator loss -mean(fake)."""

    @staticmethod
    def forward(ctx, real, fake, kind):
        ops._f32(fake, real)
        fake = fake.contiguous()
        real = real.contiguous() if real is not None else None
        loss = torch.empty((), device=fake.device, dtype=torch.float32)
        g_fake = torch.empty_like(fake)
        g_real = torch.empty_like(real) if real is not None else None
        lib().skd_adv_loss(fake.numel(), _p(real), _p(fake), kind, _p(loss), _p(g_real), _p(g_fake), _st())
        ctx.save_for_backward(g_real, g_fake)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        g_real, g_fake = ctx.saved_tensors
        return (g_real * go if g_real is not None and ctx.needs_input_grad[0] else None,
                g_fake * go if ctx.needs_input_grad[1] else None, None)


# ---------------------------------------------------------------------------------------------------- stand-alone layers
class SNConvFn(torch.autograd.Function):
    """SpectralNorm(conv).forward used on its own (networks/spectral.py:66-68): one power iteration, then
    y = conv(x, w_bar) / sigma + bias on wgmma; backward = wgmma dgrad / wgrad + the sigma term of spectral.py:34-35."""

    @staticmethod
    def forward(ctx, m, x, w_bar, bias):
        L, st = lib(), _st()
        x = ops.to_nhwc(x)
        n, cin, h, w, ldx = ops.nhwc_meta(x)
        cout, _, kh, kw = w_bar.shape
        if cin % 4 or ldx % 4 or cout % 4:
            raise ValueError("stand-alone SpectralNorm convolutions need channel counts that are multiples of 4")
        dev = x.device
        wq = ops.weight_ohwi(w_bar)
        taps = kh * kw
        s = dict(u=_f(cout, dev=dev), v=_f(taps * cin, dev=dev), sigma=_f(1, dev=dev), inv=_f(cout, dev=dev))
        L.skd_sn_power_iter(cout, taps, cin, _p(wq), _p(m.weight_u), _p(m.weight_v), _p(s["u"]), _p(s["v"]), _p(s["sigma"]), _p(s["inv"]), cout, st)
        oh, ow = ops.conv_out_hw(h, w, (kh, kw), m.stride, m.padding, m.dilation)
        y = ops.empty_nhwc(n, cout, oh, ow, dev)
        L.skd_conv2d_fwd_sm100_ex(n, h, w, cin, cout, kh, kw, m.stride, m.padding, m.dilation, _p(x), None, ldx, _p(wq), None, _p(y), cout, 0, 0,
                                  _p(s["inv"]), _p(bias), None, 0, ACT_NONE, 0.0, st)
        ctx.save_for_backward(x, w_bar, s["u"], s["v"], s["sigma"])
        ctx.m = m
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        L, st = lib(), _st()
        x, w_bar, u, v, sigma = ctx.saved_tensors
        m = ctx.m
        dy = ops.to_nhwc(dy)
        wq = ops.weight_ohwi(w_bar)
        cout, kh, kw, cin = wq.shape
        dx = dw = db = None
        if ctx.needs_input_grad[1]:
            dx = ops.conv2d_dgrad(dy, wq, tuple(x.shape), m.stride, m.padding, m.dilation) / sigma
        if ctx.needs_input_grad[2]:
            dwn = ops.conv2d_wgrad(x, dy, (kh, kw), m.stride, m.padding, m.dilation)
            dw = torch.empty_like(w_bar)
            ws = torch.zeros(L.skd_sn_weight_grad_workspace_doubles(), device=x.device, dtype=torch.float64)
            L.skd_sn_weight_grad(cout, kh * kw, cin, cin, _p(dwn), _p(wq), _p(m.weight_u), _p(m.weight_v), _p(sigma), _p(dw), 0, _p(ws), st)   # current u, v: see DiscEngine._reverse_layers
        if ctx.has_bias and ctx.needs_input_grad[3]:
            db = ops.colsum(dy)
        return None, dx, dw, db


class SelfAttnFn(torch.autograd.Function):
    """Self_Attn.forward used on its own (sagan_models.py:22-41): returns (gamma * out + x, attention)."""

    @staticmethod
    def forward(ctx, A, x, *params):
        L, st = lib(), _st()
        x = ops.to_nhwc(x)
        n_img, c, h, w, ldx = ops.nhwc_meta(x)
        if ldx != c:
            raise ValueError("Non-contiguous input")
        dev = x.device
        d = A.query_conv.out_channels
        ldq = 2 * d + c
        n = h * w
        wcat = torch.cat([A.query_conv.weight.reshape(d, c), A.key_conv.weight.reshape(d, c), A.value_conv.weight.reshape(c, c)]).contiguous()
        bias = torch.cat([A.query_conv.bias, A.key_conv.bias, A.value_conv.bias]).detach()
        qkv = _f(n_img * n, ldq, dev=dev)
        x_lo, w_lo = torch.empty_like(x), torch.empty_like(wcat)
        L.skd_split_tf32(x.numel(), _p(x), None, _p(x_lo), st)
        L.skd_split_tf32(wcat.numel(), _p(wcat), None, _p(w_lo), st)
        L.skd_conv2d_fwd_sm100_ex(1, 1, n_img * n, c, ldq, 1, 1, 1, 0, 1, _p(x), _p(x_lo), c, _p(wcat), _p(w_lo), _p(qkv), ldq, 0, 0, None, _p(bias),
                                  None, 0, ACT_NONE, 0.0, st)
        attn, o = _f(n_img, n, n, dev=dev), _f(n_img * n, c, dev=dev)
        y = ops.empty_nhwc(n_img, c, h, w, dev)
        L.skd_attn_fwd(n_img, n, c, d, _p(qkv), ldq, _p(x), _p(A.gamma), _p(attn), _p(o), _p(y), None, st)
        ctx.save_for_backward(x, qkv, attn, o, wcat)
        ctx.A = A
        ctx.mark_non_differentiable(attn)
        return y, attn

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy, _):
        L, st = lib(), _st()
        x, qkv, attn, o, wcat = ctx.saved_tensors
        A = ctx.A
        n_img, c, h, w = x.shape
        dev = x.device
        d = A.query_conv.out_channels
        ldq, n = 2 * d + c, h * w
        gy = ops.to_nhwc(gy)
        gqkv = _f(n_img * n, ldq, dev=dev)
        ggam = _f(1, dev=dev)
        wsf = _f(L.skd_attn_bwd_workspace_floats(n_img, n, c), dev=dev)
        L.skd_attn_bwd(n_img, n, c, d, _p(qkv), ldq, _p(attn), _p(o), _p(A.gamma), _p(gy), None, None, None, None, _p(gqkv), None, _p(ggam), 0,
                       _p(wsf), st)
        dw = _f(ldq, c, dev=dev)
        wsg = _f(max(L.skd_conv2d_wgrad_sm100_workspace_floats(n_img, h, w, c, ldq, 1, 1, 1, 0, 1), 4), dev=dev)
        L.skd_conv2d_wgrad_sm100(n_img, h, w, c, ldq, 1, 1, 1, 0, 1, _p(x), c, _p(gqkv), ldq, _p(dw), _p(wsg), st)
        db = _f(ldq, dev=dev)
        L.skd_colsum(n_img * n, ldq, _p(gqkv), ldq, _p(db), st)
        wt = _f(c, ldq, dev=dev)
        L.skd_weight_flip_transpose(ldq, c, 1, 1, _p(wcat), _p(wt), 0, st)
        gx = ops.empty_nhwc(n_img, c, h, w, dev)
        L.skd_conv2d_fwd_sm100_ex(1, 1, n_img * n, ldq, c, 1, 1, 1, 0, 1, _p(gqkv), None, ldq, _p(wt), None, _p(gx), c, 0, 0, None, None, _p(gy), c,
                                  ACT_NONE, 0.0, st)
        by_name = {"query_conv.weight": dw[:d].view(d, c, 1, 1), "query_conv.bias": db[:d], "key_conv.weight": dw[d:2 * d].view(d, c, 1, 1),
                   "key_conv.bias": db[d:2 * d], "value_conv.weight": dw[2 * d:].view(c, c, 1, 1), "value_conv.bias": db[2 * d:], "gamma": ggam}
        return (None, gx) + tuple(by_name[nm] for nm, _ in A.named_parameters())
