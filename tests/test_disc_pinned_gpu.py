"""The discriminator phase on the H100 against float64 with the LeakyReLU masks pinned (oracle/disc_pinned.py), and the kernel paths
of csrc/disc.cu that only the whole-discriminator tests reached before.

Whole phase.  NetModel's discriminator sequence runs through the public surfaces (Discriminator, CriterionAdvForG, CriterionAdv,
CriterionAdditionalGP with injected alpha): the generator pass -mean D(xs) with d / d xs, fresh gradients, D(xt), D(xs), the
adversarial loss (+ the penalty) and backward.  Every call of the engine's forward records the masks it chose, h[:B] > 0 per SN
layer (the criterion of the mask and un-shuffle kernels), and the float64 oracle replays the sequence with those masks, so both
evaluate the same smooth piece of the network: first and second derivatives agree up to fp32 rounding, and the tolerances are
fp32-grade instead of the 2e-2 that mask flips force on the unpinned comparisons (tests/test_discriminator_gpu.py).  The pinning
cannot hide a forward bug: a separate guard runs the unpinned float64 forward and requires every element where the GPU's mask
disagrees with its sign to lie within rounding distance of zero.

Tolerances (rel-L2 unless stated) are the worst values measured on an H100 80GB HBM3 (700 W power limit) with a margin of 3-4x;
the per-quantity worst values are in DESIGN.md §4.
  * fp32-grade, 3e-5 (worst 8.4e-6, the attention gamma): outputs, attention maps, losses (against the outputs' magnitude), penalty
    and norms, d / d xs, BN gamma / beta, attention gamma, every bias, the last convolution's weight (SIMT fp32), u / v and the BN
    running statistics;
  * TF32, 1.5e-3 (worst 4.4e-4): the SN convolutions' weight_bar and the q / k / v weights, whose weight-gradient GEMMs are
    single-pass TF32;
  * gradients that cancel analytically (attn2.value_conv.bias) in absolute terms against the largest gradient norm, 3e-8 (worst 6.9e-9).
The mask guard allows a disagreement at |z| <= 1e-5 rms(z) of its layer; the largest seen was 1.7e-7, at most one per call.
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_tf32_rounding_cpu import split_tf32

pytestmark = pytest.mark.gpu

TOL = dict(fp32=3e-5, tf32=1.5e-3, cancel=3e-8)        # measured worst: 8.4e-6, 4.4e-4, 6.9e-9
MASK_TAU = 1e-5            # |z| / rms(z) of the layer below which a mask disagreement counts as rounding (measured worst: 1.7e-7)


def rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rn_tf32(t):
    """cvt.rn.tf32.f32: round to nearest even at 10 mantissa bits"""
    u = t.contiguous().view(torch.int32)
    return ((u + 0x0FFF + ((u >> 13) & 1)) & ~0x1FFF).view(torch.float32)


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.fixture(scope="module")
def L():
    from structure_knowledge_distillation_b200._cabi import lib
    return lib()


# ------------------------------------------------------------------------------------------------ whole discriminator phase
def _port_state(mode, cin):
    from oracle import port
    torch.manual_seed(11)
    Dp = port.Discriminator(mode, cin, 64)
    with torch.no_grad():
        Dp.attn1.gamma.fill_(-0.4); Dp.attn2.gamma.fill_(0.25)            # gamma = 0 would hide the attention path
        if mode == 1:
            Dp.preprocess_additional.weight.mul_(1.2)
    return {k: v.clone() for k, v in Dp.state_dict().items()}


def _inputs(mode, B, C, H, W, g):
    xt = torch.randn(B, C, H, W, device="cuda", generator=g) * 3
    xs = torch.randn(B, C, H, W, device="cuda", generator=g) * 3
    if mode == 3:                                                   # the rescale mode's range
        xs = torch.rand(B, C, H, W, device="cuda", generator=g) * 255
    alpha = torch.rand(B, 1, 1, 1, device="cuda", generator=g)
    return xs, xt, alpha


def _is_tf32_weight(name):
    return name.endswith(".weight_bar") or name.endswith(("query_conv.weight", "key_conv.weight", "value_conv.weight"))


#   name            B   H    W  classes adv       mode split_k   what it reaches
PHASES = [
    ("bench",       8, 65, 129, 19, "wgan-gp", 1, True),   # the benchmark step
    ("bench_nosk",  8, 65, 129, 19, "wgan-gp", 1, False),  # the same without split-K convolutions
    ("bench_hinge", 8, 65, 129, 19, "hinge",   1, True),   # hinge masks
    ("cfg4",       16, 46,  61, 19, "wgan-gp", 1, True),   # 2x3 top under the size-aware head
    ("crop769",     2, 97,  97, 19, "wgan-gp", 1, True),   # attn1 over 144 positions (row-stripe kernels)
    ("batch1",      1, 65, 129, 19, "wgan-gp", 1, True),   # the rank-one sigma term as large as the rest of l4's gradient
    ("voc",         4, 65, 129, 21, "wgan-gp", 1, True),   # Cin 21 padded to 24
    ("tanh",        2, 65, 129, 19, "wgan-gp", 2, True),
    ("tanh_hinge",  2, 65, 129, 19, "hinge",   2, True),
    ("rescale",     2, 65, 129, 19, "wgan-gp", 3, True),
    ("rescale_hinge", 2, 65, 129, 19, "hinge", 3, True),
]


@pytest.mark.parametrize("case", PHASES, ids=[c[0] for c in PHASES])
def test_discriminator_phase_vs_pinned_float64(case):
    from oracle import disc_pinned
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.utils.criterion import CriterionAdditionalGP, CriterionAdv, CriterionAdvForG
    name, B, H, W, C, adv, mode, split_k = case
    state = _port_state(mode, C)
    D = Discriminator(mode, C, B, 65, 64).cuda().train()
    D.load_state_dict(state, strict=True)
    D.engine.split_k = split_k
    Dq = disc_pinned.PinnedDiscriminator(mode, C, 64)
    Dq.load_state_dict(state, strict=True)
    Dq = Dq.cuda().double().train()
    Du = copy.deepcopy(Dq)                                            # unpinned, for the mask guard
    xs, xt, alpha = _inputs(mode, B, C, H, W, _gen(H * W + C + 7 * mode + len(adv)))

    # ---- GPU: the engine's forward records the masks it chose, h[:B] > 0 per SN layer, at every call
    calls = []
    forward = D.engine.forward

    def recording_forward(x, *args, **kwargs):
        t = forward(x, *args, **kwargs)
        calls.append(dict(tape=t, masks=[(h[:t.B] > 0).permute(0, 3, 1, 2).contiguous() for h in t.h]))
        return t
    D.engine.forward = recording_forward
    xs_g = xs.clone().requires_grad_(True)
    o_g = D(xs_g)
    loss_g = CriterionAdvForG(adv)(o_g, None)
    loss_g.backward()
    for p in D.parameters():
        p.grad = None
    o_t, o_s = D(xt), D(xs)                                           # kd_model.py's order
    loss = CriterionAdv(adv)(o_s, o_t)
    gp = None
    if adv == "wgan-gp":
        crit = CriterionAdditionalGP(D, 10.0)
        crit.alpha = alpha
        gp = crit([xs], [xt])
        loss = loss + gp
    loss.backward()
    torch.cuda.synchronize()
    assert len(calls) == (4 if adv == "wgan-gp" else 3)
    hinge = (1.0 - o_t[0].detach() > 0, 1.0 + o_s[0].detach() > 0) if adv == "hinge" else None

    # ---- float64 on the same smooth piece
    Dq.pin([c["masks"] for c in calls])
    ref = disc_pinned.discriminator_phase(Dq, xs.double(), xt.double(), adv, alpha.double(), 10.0, hinge)

    # ---- mask guard: every disagreement with the unpinned float64 pre-activation's sign lies within rounding distance of zero
    with torch.no_grad():
        Du(xs.double()); Du(xt.double()); Du(xs.double())
        if adv == "wgan-gp":
            a = alpha.double()
            Du(a * xt.double() + (1 - a) * xs.double())
    flips, worst_flip = [], 0.0
    for c, pre in zip(calls, Du.preacts):
        per_call = 0
        for m, z in zip(c["masks"], pre):
            dis = m != (z > 0)
            per_call += int(dis.sum())
            if bool(dis.any()):
                ratio = float(z[dis].abs().max() / z.pow(2).mean().sqrt())
                worst_flip = max(worst_flip, ratio)
        flips.append(per_call)

    # ---- compare
    err = {}
    out_scale = float(torch.stack([o[0].detach().abs().mean() for o in ref["outs"]]).max())
    for c, (mine, theirs) in enumerate(zip((o_g, o_t, o_s), ref["outs"])):
        for k, key in enumerate(("out", "p1", "p2")):
            err["%s%d" % (key, c)] = rel(mine[k], theirs[k])
    # losses are means of outputs of both signs: their rounding is measured against the outputs' magnitude
    err["loss_g"] = abs(float(loss_g) - float(ref["loss_g"])) / max(abs(float(ref["loss_g"])), out_scale)
    err["loss"] = abs(float(loss) - float(ref["loss"])) / max(abs(float(ref["loss"])), out_scale)
    if gp is not None:
        err["gp"] = rel(gp, ref["gp"])
        err["norms"] = rel(calls[-1]["tape"].norms, ref["norms"])
    err["xs_grad"] = rel(xs_g.grad, ref["xs_grad"])
    grads = {n: p.grad for n, p in D.named_parameters() if p.requires_grad}
    assert sorted(grads) == sorted(ref["grads"])
    top = max(float(g.norm()) for g in ref["grads"].values())
    groups = dict(fp32={}, tf32={}, cancel={})
    for n, g in ref["grads"].items():
        assert grads[n] is not None, n
        if float(g.norm()) < 1e-5 * top:
            groups["cancel"][n] = float((grads[n].double().cpu() - g.cpu()).norm()) / top
        else:
            groups["tf32" if _is_tf32_weight(n) else "fp32"][n] = rel(grads[n], g)
    sd, sq = D.state_dict(), Dq.state_dict()
    for n, t in sq.items():
        if n.endswith(("weight_u", "weight_v", "running_mean", "running_var")):
            err[n] = rel(sd[n], t)
        elif n.endswith("num_batches_tracked"):
            assert int(sd[n]) == int(t) == len(calls), n
    groups["fp32"].update(err)
    worst = {k: max(v.items(), key=lambda kv: kv[1]) if v else ("-", 0.0) for k, v in groups.items()}
    print("\nPARITY disc_pinned %s B=%d %dx%d C=%d %s mode %d split_k %d: mask disagreements per call %s (worst |z|/rms %.1e); "
          "worst fp32 %.2e (%s), tf32 %.2e (%s), cancelling %.2e (%s)" %
          (name, B, H, W, C, adv, mode, split_k, flips, worst_flip, worst["fp32"][1], worst["fp32"][0], worst["tf32"][1],
           worst["tf32"][0], worst["cancel"][1], worst["cancel"][0]))
    print("PARITY disc_pinned %s all %s" % (name, {k: "%.1e" % v for g in groups.values() for k, v in g.items()}))
    assert worst_flip <= MASK_TAU, (worst_flip, flips)
    for k, v in groups.items():
        bad = {n: e for n, e in v.items() if not e <= TOL[k]}
        assert not bad, (k, bad)


# ------------------------------------------------------------------------------------------------ BatchNorm2d at the step's P
def _bn_x(layout, B, C, H, W, Cp, g):
    if layout == "nchw":
        return torch.randn(B, C, H, W, device="cuda", generator=g) * 2 + 0.3
    if layout == "channels_last":
        return (torch.randn(B, C, H, W, device="cuda", generator=g) * 2 + 0.3).contiguous(memory_format=torch.channels_last)
    return (torch.randn(B, H, W, Cp, device="cuda", generator=g) * 2 + 0.3).permute(0, 3, 1, 2)[:, :C]     # nhwc, pitch Cp


@pytest.fixture(scope="module")
def bn_ws(L):
    """one workspace for every case: its self-resetting block counter must survive calls of any shape back to back"""
    return torch.zeros(L.skd_bn2d_workspace_doubles(), device="cuda", dtype=torch.float64)


@pytest.mark.parametrize("layout,B,C,H,W,Cp", [("nchw", 8, 19, 65, 129, 20), ("channels_last", 8, 19, 65, 129, 20),
                                               ("nhwc", 8, 19, 65, 129, 20), ("nchw", 16, 19, 46, 61, 20),
                                               ("nhwc", 2, 21, 97, 97, 24), ("nchw", 1, 19, 65, 129, 20)])
def test_bn2d_first_and_second_order_at_step_shapes(L, bn_ws, layout, B, C, H, W, Cp):
    """stats (x3) -> apply with out_lo -> reduce(a) -> reduce(a, b2) -> Jacobian (strided, and dense with out_lo) -> param_grad in
    first order (accumulate 0) and second order (sums_t / sums_v, accumulate 1), against float64: BatchNorm2d and autograd, and for
    the second order torch.func.jvp of BatchNorm along xdot then autograd of <gth, tangent> with respect to gamma."""
    from structure_knowledge_distillation_b200 import ops
    g = _gen(B * H * W + C)
    P, eps, mom = B * H * W, 1e-5, 0.1
    xsl = [_bn_x(layout, B, C, H, W, Cp, g) for _ in range(3)]
    rm, rv = torch.randn(C, device="cuda", generator=g) * 0.1, torch.rand(C, device="cuda", generator=g) + 0.5
    rm_d, rv_d = rm.double(), rv.double()
    nbt = torch.zeros((), device="cuda", dtype=torch.int64)
    mean, rstd = torch.empty(32, device="cuda"), torch.empty(32, device="cuda")
    for x in xsl:
        L.skd_bn2d_stats(B, C, H * W, _p(x), *ops.pixel_strides(x), eps, mom, _p(rm), _p(rv), _p(nbt), _p(mean), _p(rstd), _p(bn_ws), _st())
        xd = x.double()
        mu, var = xd.mean((0, 2, 3)), xd.var((0, 2, 3), unbiased=False)
        rm_d, rv_d = (1 - mom) * rm_d + mom * mu, (1 - mom) * rv_d + mom * var * P / (P - 1)
    x, xd = xsl[-1], xsl[-1].double()
    err = dict(mean=rel(mean[:C], mu), rstd=rel(rstd[:C], (var + eps).rsqrt()), running_mean=rel(rm, rm_d), running_var=rel(rv, rv_d))
    assert int(nbt) == 3
    xs_ = ops.pixel_strides(x)
    gam, bet = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    gam_d, bet_d = gam.double().requires_grad_(True), bet.double().requires_grad_(True)

    def bn(t):
        return F.batch_norm(t, None, None, gam_d, bet_d, training=True, eps=eps)
    dense = lambda t: t[..., :C].permute(0, 3, 1, 2).double()       # [B][H][W][Cp] rows -> NCHW float64
    # apply: dense rows, zero pad channels, exact TF32 lo part
    out, out_lo = torch.full((B, H, W, Cp), 7.0, device="cuda"), torch.full((B, H, W, Cp), 7.0, device="cuda")
    L.skd_bn2d_apply(B, C, H * W, _p(x), *xs_, _p(mean), _p(rstd), _p(gam), _p(bet), _p(out), _p(out_lo), Cp, _st())
    xhat = (xd - mu.view(1, C, 1, 1)) * (var + eps).rsqrt().view(1, C, 1, 1)
    err["apply"] = rel(dense(out), bn(xd))
    assert float(out[..., C:].abs().max()) == 0.0 and torch.equal(_bits(out_lo), _bits(_rn_tf32(out - _rn_tf32(out))))
    # adjoints / tangent as the engine holds them: dense [P][Cp] rows, pad channels not read (filled with large values here);
    # xdot and gth lean on xhat so that every term of the second-order formula carries weight
    pad = lambda t: torch.cat([t.permute(0, 2, 3, 1), torch.full((B, H, W, Cp - C), 1e6, device="cuda")], 3).contiguous()
    nchw = lambda: torch.randn(B, C, H, W, device="cuda", generator=g)
    gh = pad(nchw())
    xdot = pad(nchw() + 0.5 * xhat.float())
    gth = pad(nchw() - 0.7 * xhat.float())
    sums_g, sums_t, sums_v = (torch.full((96,), 7.0, device="cuda") for _ in range(3))
    L.skd_bn2d_reduce(B, C, H * W, _p(x), *xs_, _p(mean), _p(rstd), _p(gh), None, Cp, _p(sums_g), _p(bn_ws), _st())
    L.skd_bn2d_reduce(B, C, H * W, _p(x), *xs_, _p(mean), _p(rstd), _p(gth), _p(xdot), Cp, _p(sums_t), _p(bn_ws), _st())
    L.skd_bn2d_reduce(B, C, H * W, _p(x), *xs_, _p(mean), _p(rstd), _p(xdot), None, Cp, _p(sums_v), _p(bn_ws), _st())
    S = lambda t: t.sum((0, 2, 3))
    err["sums_g"] = rel(torch.cat([sums_g[:C], sums_g[32:32 + C]]), torch.cat([S(dense(gh)), S(dense(gh) * xhat)]))
    err["sums_t"] = rel(torch.cat([sums_t[:C], sums_t[32:32 + C], sums_t[64:64 + C]]),
                        torch.cat([S(dense(gth)), S(dense(gth) * xhat), S(dense(gth) * dense(xdot))]))
    err["sums_v"] = rel(torch.cat([sums_v[:C], sums_v[32:32 + C]]), torch.cat([S(dense(xdot)), S(dense(xdot) * xhat)]))
    assert float(sums_g[64:64 + C].abs().max()) == 0.0                 # b2 = NULL: the third product is zero
    # float64 references: y, the tangent along xdot, d/dx of <gh, y>, and the parameter gradients of both orders
    xr = xd.clone().requires_grad_(True)
    y = bn(xr)
    gx_ref, g1_gam, g1_bet = torch.autograd.grad(y, [xr, gam_d, bet_d], dense(gh), retain_graph=True)
    _, tangent = torch.func.jvp(bn, (xd,), (dense(xdot),))
    (g2_gam,) = torch.autograd.grad((y * dense(gh)).sum() + (tangent * dense(gth)).sum(), [gam_d])
    # Jacobian in x's own layout (the input gradient) and dense with lo part (the penalty's tangent into layer 1)
    dx = torch.empty_strided(x.shape, x.stride(), device="cuda")
    L.skd_bn2d_jacobian(B, C, H * W, _p(x), *xs_, _p(mean), _p(rstd), _p(gam), _p(gh), Cp, _p(sums_g), _p(dx), *ops.pixel_strides(dx), C, None, _st())
    err["jacobian_strided"] = rel(dx, gx_ref)
    tj, tj_lo = torch.full((B, H, W, Cp), 7.0, device="cuda"), torch.full((B, H, W, Cp), 7.0, device="cuda")
    L.skd_bn2d_jacobian(B, C, H * W, _p(x), *xs_, _p(mean), _p(rstd), _p(gam), _p(xdot), Cp, _p(sums_v), _p(tj), H * W * Cp, 1, Cp, Cp,
                        _p(tj_lo), _st())
    err["jacobian_dense"] = rel(dense(tj), tangent)
    assert float(tj[..., C:].abs().max()) == 0.0 and torch.equal(_bits(tj_lo), _bits(_rn_tf32(tj - _rn_tf32(tj))))
    dgam, dbet = torch.full((C,), 7.0, device="cuda"), torch.full((C,), 7.0, device="cuda")
    L.skd_bn2d_param_grad(C, P, _p(rstd), _p(sums_g), None, None, _p(dgam), _p(dbet), 0, _st())
    err["dgamma_1"], err["dbeta_1"] = rel(dgam, g1_gam), rel(dbet, g1_bet)
    L.skd_bn2d_param_grad(C, P, _p(rstd), _p(sums_g), _p(sums_t), _p(sums_v), _p(dgam), _p(dbet), 1, _st())
    err["dgamma_2"], err["dbeta_2"] = rel(dgam, g1_gam + g2_gam), rel(dbet, 2 * g1_bet)
    print("\nPARITY bn2d %s B=%d C=%d %dx%d Cp=%d" % (layout, B, C, H, W, Cp), {k: "%.1e" % v for k, v in err.items()})
    bad = {k: v for k, v in err.items() if not v < 1e-5}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ LeakyReLU mask multiply
def _engine_lengths(B, H, W):
    out, hc, wc = [], H, W
    for cout in (64, 128, 256, 512):
        hc, wc = (hc - 2) // 2 + 1, (wc - 2) // 2 + 1
        out.append(B * hc * wc * cout)
    return out


@pytest.mark.parametrize("layer", [0, 1, 2, 3])
def test_mask_mul_bit_exact_at_engine_lengths(L, layer):
    """out = in * leaky'(ref) at the benchmark step's lengths: first order (period == n) and the joint [primal | tangent] form
    (period == n / 2: the tangent half takes the primal mask), with +0, -0, negatives, positive denormals and NaN in ref."""
    per = _engine_lengths(8, 65, 129)[layer]
    g = _gen(per)
    ref = torch.randn(per, device="cuda", generator=g)
    special = torch.tensor([0.0, -0.0, -1.0, -1e-30, 1e-40, 1.4e-45, -1e-40, float("nan"), -float("nan"), 3.0], device="cuda")
    where = torch.randint(0, per, (per // 50,), device="cuda", generator=g)
    ref[where] = special[torch.randint(0, len(special), (len(where),), device="cuda", generator=g)]
    slope = torch.tensor(0.1, dtype=torch.float32)
    for n, with_lo in ((per, True), (2 * per, False), (2 * per, True)):
        v = torch.randn(n, device="cuda", generator=g)
        out, lo = torch.full_like(v, 7.0), torch.full_like(v, 7.0)
        L.skd_disc_mask_mul(n, per, _p(ref), _p(v), _p(out), _p(lo) if with_lo else None, 0.1, _st())
        rep = ref.repeat(n // per)
        want = torch.where(rep > 0, v, v * slope.cuda())
        assert torch.equal(_bits(out), _bits(want)), (n, with_lo)
        if with_lo:
            assert torch.equal(_bits(lo), _bits(_rn_tf32(out - _rn_tf32(out))))
        else:
            assert bool((lo == 7.0).all())


def test_mask_mul_rejects_lengths_off_the_vector_width(L):
    buf = torch.zeros(64, device="cuda")
    out = torch.full((64,), 7.0, device="cuda")
    for n, period in ((6, 6), (8, 6), (10, 8)):
        before = L.skd_kernel_launches()
        with pytest.raises(RuntimeError, match="skd_disc_mask_mul"):
            L.skd_disc_mask_mul(n, period, _p(buf), _p(buf), _p(out), None, 0.1, _st())
        assert L.skd_kernel_launches() == before
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


# ------------------------------------------------------------------------------------------------ weight staging
@pytest.mark.parametrize("rows,cin", [(64 * 16, 11), (64 * 16, 19), (64 * 16, 21), (128 * 16, 64), (256 * 16, 128), (512 * 16, 256),
                                      (32, 256), (256, 256), (64, 512), (512, 512)])
def test_weight_prep_bit_exact(L, rows, cin):
    """SN layer weights [Cout * 16 taps][Cin] (Cin 11 = CamVid, 19 = Cityscapes, 21 = VOC) and the q / k / v rows of attn1 / attn2:
    a channel-padded copy with zero pad channels and the TF32 lo part of exactly that copy."""
    g = _gen(rows + cin)
    w = torch.randn(rows, cin, device="cuda", generator=g) * 0.1
    w.view(-1)[:4] = torch.tensor([1e-40, -0.0, 2.0 ** -20 * 1.5, 3.0], device="cuda")
    cin_p = (cin + 3) // 4 * 4
    wp, wlo = torch.full((rows, cin_p), 7.0, device="cuda"), torch.full((rows, cin_p), 7.0, device="cuda")
    L.skd_disc_weight_prep(rows, cin, cin_p, _p(w), _p(wp), _p(wlo), _st())
    assert torch.equal(_bits(wp[:, :cin]), _bits(w)) and torch.equal(_bits(wp[:, cin:]), torch.zeros_like(_bits(wp[:, cin:])))
    _, lo_ref = split_tf32(wp.cpu().numpy())
    assert np.array_equal(wlo.cpu().numpy().view(np.uint32), lo_ref.view(np.uint32))


# ------------------------------------------------------------------------------------------------ WGAN-GP reductions
@pytest.mark.parametrize("length", [65 * 129 * 20, 46 * 61 * 20, 97 * 97 * 24])
@pytest.mark.parametrize("B", [1, 8, 16])
def test_gp_norms_and_direction(L, B, length):
    g = _gen(B * 7 + length)
    u = torch.rand(B, 1, device="cuda", generator=g)
    scale = torch.where(torch.arange(B, device="cuda").view(B, 1) % 2 == 0, 0.2 + 0.5 * u, 1.3 + 0.7 * u)     # norms away from 1
    gv = torch.randn(B, length, device="cuda", generator=g) / length ** 0.5 * scale
    norms, gpl = torch.empty(B, device="cuda"), torch.empty((), device="cuda")
    L.skd_gp_norms(B, length, _p(gv), 10.0, _p(norms), _p(gpl), _st())
    gd = gv.double().requires_grad_(True)
    nd = gd.norm(dim=1)
    ref = 10.0 * ((nd - 1) ** 2).mean()
    (dref,) = torch.autograd.grad(ref, gd)
    assert rel(norms, nd) < 1e-6 and rel(gpl, ref) < 1e-5
    for up in (None, torch.tensor(0.37, device="cuda")):
        v = torch.full_like(gv, 7.0)
        L.skd_gp_direction(B, length, _p(gv), _p(norms), 10.0, _p(up), _p(v), _st())
        assert rel(v, dref * (1.0 if up is None else 0.37)) < 1e-5


# ------------------------------------------------------------------------------------------------ adversarial losses
@pytest.mark.parametrize("n", [1, 40, 96, 1500])
def test_adv_loss_all_kinds_and_hinge_kinks(L, n):
    """One 128-thread block (1500 runs its strided loop): the loss against float64; the gradients bit-equal to torch autograd's
    in fp32, with real = 1 and fake = -1 exactly at the hinge's kinks, where autograd's relu gradient is 0."""
    g = _gen(n)
    real, fake = torch.randn(n, device="cuda", generator=g) * 2, torch.randn(n, device="cuda", generator=g) * 2
    real[::3], fake[1::3] = 1.0, -1.0
    fns = {0: lambda r, f: -r.mean() + f.mean(), 1: lambda r, f: F.relu(1 - r).mean() + F.relu(1 + f).mean(), 2: lambda r, f: -f.mean()}
    for kind, fn in fns.items():
        loss, gr, gf = torch.empty((), device="cuda"), torch.full((n,), 7.0, device="cuda"), torch.full((n,), 7.0, device="cuda")
        L.skd_adv_loss(n, _p(real), _p(fake), kind, _p(loss), _p(gr), _p(gf), _st())
        ref = fn(real.double(), fake.double())
        scale = float(real.double().abs().mean() + fake.double().abs().mean() + 1.0)
        assert abs(float(loss) - float(ref)) <= 1e-6 * scale, (kind, float(loss), float(ref))
        r32, f32 = real.clone().requires_grad_(True), fake.clone().requires_grad_(True)
        gr_ref, gf_ref = torch.autograd.grad(fn(r32, f32), [r32, f32], allow_unused=True)
        assert torch.equal(gf, gf_ref), kind
        assert torch.equal(gr, gr_ref if gr_ref is not None else torch.zeros_like(gr)), kind


# ------------------------------------------------------------------------------------------------ the last convolution
@pytest.mark.parametrize("top", [(4, 8), (2, 3), (6, 6)])
def test_last_conv_tops_ones_and_accumulate(L, top):
    """4x8 top (the benchmark), 2x3 (size-aware window) and 6x6 (a 3x3 output); the penalty's ones as gout (NULL) and a given
    gout; the weight and bias gradients accumulated onto existing values."""
    hh, ww = top
    B, C = 3, 512
    kh, kw = min(4, hh), min(4, ww)
    oh, ow = hh - kh + 1, ww - kw + 1
    g = _gen(hh * ww)
    x = torch.randn(B, hh, ww, C, device="cuda", generator=g)
    w = torch.randn(1, 4, 4, C, device="cuda", generator=g) * 0.05
    bias = torch.tensor([0.2], device="cuda")
    out = torch.empty(B, oh, ow, device="cuda")
    L.skd_disc_last_fwd(B, hh, ww, C, kh, kw, _p(x), _p(w), 4 * C, _p(bias), _p(out), _st())
    xd = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    wd = w[:, :kh, :kw].permute(0, 3, 1, 2).double().requires_grad_(True)
    ref = F.conv2d(xd, wd, bias.double())
    assert rel(out, ref) < 1e-5
    for gout in (None, torch.randn(B, oh, ow, device="cuda", generator=g)):
        go = torch.ones(B, 1, oh, ow, device="cuda", dtype=torch.float64) if gout is None else gout.double().view(B, 1, oh, ow)
        gx_ref, gw_ref = torch.autograd.grad(ref, [xd, wd], go, retain_graph=True)
        gx = torch.full_like(x, 7.0)
        L.skd_disc_last_dgrad(B, hh, ww, C, kh, kw, _p(gout), _p(w), 4 * C, _p(gx), None, _st())
        assert rel(gx.permute(0, 3, 1, 2), gx_ref) < 1e-5
        gw0, gb0 = torch.randn(1, 4, 4, C, device="cuda", generator=g), torch.randn(1, device="cuda", generator=g)
        gw, gb = gw0.clone(), gb0.clone()
        L.skd_disc_last_wgrad(B, hh, ww, C, kh, kw, _p(x), _p(gout), _p(gw), 4 * C, _p(gb), 1, _st())
        assert rel(gw[:, :kh, :kw].permute(0, 3, 1, 2) - gw0[:, :kh, :kw].permute(0, 3, 1, 2), gw_ref) < 1e-5
        assert torch.equal(gw[:, kh:], gw0[:, kh:]) and torch.equal(gw[:, :, kw:], gw0[:, :, kw:])      # outside the window: untouched
        assert abs(float(gb - gb0) - float(go.sum())) <= 1e-5 * float(go.abs().sum())
