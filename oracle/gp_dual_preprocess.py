"""The "reverse over forward" WGAN-GP parameter gradient of oracle/gp_dual.py for the discriminator's parameter-free input modes
(TEST INFRASTRUCTURE ONLY): preprocess_GAN_mode 2 (tanh) and 3 (2 (x / 255 - 0.5)), networks/sagan_models.py:149-152.

Same operation sequence as gp_dual.gp_and_param_grads, which states mode 1 (batch-statistics BatchNorm2d), with the input map
replaced: h = f(x) with the diagonal Jacobian J = f'(x).  The penalty's x is detached (utils/criterion.py:109-110), so J is a
constant of the parameters:
  * the input gradient is g = J * (d(sum out) / dh);
  * the tangent along v enters the first convolution as J * v;
  * the joint reverse pass ends at layer 1's weight gradient -- there is no preprocessing parameter and no second-order term.
This is what networks/sagan_engine.py does in these modes; tests/test_disc_preprocess_cpu.py pins it against torch's double
backward of oracle/port.py in float64.
"""
import torch
import torch.nn.functional as F

from .gp_dual import LEAK, _Attn, _maps, _rows, attn_forward, attn_joint_backward, attn_tangent, power_iteration, sn_weight_grad


def pointwise_prep(mode, x):
    """-> (h, J): the mode's map and its diagonal Jacobian at x."""
    if mode == 2:
        h = torch.tanh(x)
        return h, 1 - h * h
    if mode == 3:
        return 2 * (x / 255 - 0.5), torch.full_like(x, 2.0 / 255)
    raise ValueError("preprocess mode 2 (tanh) or 3 (rescale) only; mode 1 is oracle/gp_dual.py")


def _dgrad(gz, L, like):
    op = (like.shape[2] - ((gz.shape[2] - 1) * L["s"] - 2 * L["p"] + 4), like.shape[3] - ((gz.shape[3] - 1) * L["s"] - 2 * L["p"] + 4))
    return F.conv_transpose2d(gz, L["wn"], None, L["s"], L["p"], output_padding=op)


def gp_and_param_grads(D, x, lambda_gp):
    """GP value and d(GP)/d(theta) for oracle/port.Discriminator `D` in mode 2 or 3 (imsize-65 branch) at the interpolated input x
    (B,19,H,W), AFTER one power iteration per SN layer (the caller's D(x) would do the same).
    Returns (gp, grads: dict name -> tensor with the state-dict names of the trainable parameters)."""
    dt = x.dtype
    B = x.shape[0]
    # ---- power iteration (state advances, like a forward call)
    st = []
    for sn in (D.l1[0], D.l2[0], D.l3[0], D.l4[0]):
        m = sn.module
        u, v, sigma = power_iteration(m.weight_bar.detach().to(dt), m.weight_u.detach().to(dt), m.weight_v.detach().to(dt))
        m.weight_u.data = u.to(m.weight_u.dtype); m.weight_v.data = v.to(m.weight_v.dtype)
        st.append(dict(w=m.weight_bar.detach().to(dt), b=m.bias.detach().to(dt), u=u, v=v, sigma=sigma,
                       wn=m.weight_bar.detach().to(dt) / sigma, s=sn.stride, p=sn.padding))
    at = [_Attn(D.attn1), _Attn(D.attn2)]
    for a in at:
        a.w, a.b, a.gamma = a.w.to(dt), a.b.to(dt), a.gamma.to(dt)
    w5, b5 = D.last[0].weight.detach().to(dt), D.last[0].bias.detach().to(dt)

    # ---- 1. primal forward
    h, jac = pointwise_prep(D.mode, x)
    acts, zs, att = [h], [], {}
    for i, L in enumerate(st):
        z = F.conv2d(acts[-1], L["wn"], L["b"], L["s"], L["p"])
        zs.append(z)
        h = F.leaky_relu(z, LEAK)
        if i in (2, 3):
            A = at[i - 2]
            xr = _rows(h)
            q, k, v = A.split(xr @ A.w.t() + A.b)
            y, a, o = attn_forward(q, k, v, xr, A.gamma)
            att[i] = dict(x=xr, q=q, k=k, v=v, a=a, o=o, like=h)
            h = _maps(y, h)
        acts.append(h)
    out = F.conv2d(acts[-1], w5, b5)

    # ---- 2. first-order chain to the input: g = J * d(sum out)/dh
    gh = F.conv_transpose2d(torch.ones_like(out), w5)
    for i in (3, 2, 1, 0):
        if i in (2, 3):
            A, T = at[i - 2], att[i]
            gq, gk, gv, gx, _, _, _, _, _ = attn_joint_backward(T["q"], T["k"], T["v"], T["a"], T["o"], A.gamma, _rows(gh))
            gh = _maps(torch.cat([gq, gk, gv], -1) @ A.w + gx, T["like"])
        gh = _dgrad(gh * torch.where(zs[i] > 0, 1.0, LEAK), st[i], acts[i])
    g = jac * gh
    gn = g.flatten(1).norm(dim=1)
    gp = lambda_gp * ((gn - 1) ** 2).mean()
    vdir = (2 * lambda_gp / B * (gn - 1) / gn).view(B, 1, 1, 1) * g            # constant tangent direction

    # ---- 3. tangent forward along v
    tacts, tatt = [jac * vdir], {}
    for i, L in enumerate(st):
        th = F.conv2d(tacts[-1], L["wn"], None, L["s"], L["p"]) * torch.where(zs[i] > 0, 1.0, LEAK)
        if i in (2, 3):
            A, T = at[i - 2], att[i]
            txr = _rows(th)
            tq, tk, tv = A.split(txr @ A.w.t())                                # no bias in the tangent
            ty, ds, da, do = attn_tangent(T["q"], T["k"], T["v"], T["a"], tq, tk, tv, txr, A.gamma)
            tatt[i] = dict(x=txr, q=tq, k=tk, v=tv, ds=ds, da=da, do=do)
            th = _maps(ty, T["like"])
        tacts.append(th)

    # ---- 4. reverse pass over the joint graph: adjoint of sum(tangent out) w.r.t. theta
    grads = {}
    ones = torch.ones_like(out)
    grads["last.0.weight"] = torch.nn.grad.conv2d_weight(tacts[-1], w5.shape, ones)
    grads["last.0.bias"] = torch.zeros_like(b5)
    gth = F.conv_transpose2d(ones, w5)                           # adjoint of the tangent activation
    gh = torch.zeros_like(gth)                                   # adjoint of the primal activation
    for i, name in zip((3, 2, 1, 0), ("l4", "l3", "l2", "l1")):
        if i in (2, 3):
            A, T, TT = at[i - 2], att[i], tatt[i]
            gq, gk, gv, gx, gg, gtq, gtk, gtv, gtx = attn_joint_backward(
                T["q"], T["k"], T["v"], T["a"], T["o"], A.gamma, _rows(gh), TT["q"], TT["k"], TT["v"], TT["ds"], TT["da"], TT["do"],
                _rows(gth))
            gqkv, gtqkv = torch.cat([gq, gk, gv], -1), torch.cat([gtq, gtk, gtv], -1)
            gw = gqkv.flatten(0, 1).t() @ T["x"].flatten(0, 1) + gtqkv.flatten(0, 1).t() @ TT["x"].flatten(0, 1)
            gb = gqkv.sum((0, 1))
            pre = "attn1." if i == 2 else "attn2."
            d, c = A.d, A.c
            grads[pre + "query_conv.weight"] = gw[:d].reshape(d, c, 1, 1); grads[pre + "query_conv.bias"] = gb[:d]
            grads[pre + "key_conv.weight"] = gw[d:2 * d].reshape(d, c, 1, 1); grads[pre + "key_conv.bias"] = gb[d:2 * d]
            grads[pre + "value_conv.weight"] = gw[2 * d:].reshape(c, c, 1, 1); grads[pre + "value_conv.bias"] = gb[2 * d:]
            grads[pre + "gamma"] = gg.reshape(1)
            gh = _maps(gqkv @ A.w + gx, T["like"])
            gth = _maps(gtqkv @ A.w + gtx, T["like"])
        mask = torch.where(zs[i] > 0, 1.0, LEAK)
        gz, gtz = gh * mask, gth * mask
        L = st[i]
        d_wn = torch.nn.grad.conv2d_weight(acts[i], L["w"].shape, gz, L["s"], L["p"]) + \
            torch.nn.grad.conv2d_weight(tacts[i], L["w"].shape, gtz, L["s"], L["p"])
        grads[name + ".0.module.weight_bar"] = sn_weight_grad(d_wn, L["w"], L["u"], L["v"], L["sigma"])
        grads[name + ".0.module.bias"] = gz.sum((0, 2, 3))
        if i > 0:                                                # layer 1's data gradient feeds no parameter
            gh, gth = _dgrad(gz, L, acts[i]), _dgrad(gtz, L, acts[i])
    return gp, grads
