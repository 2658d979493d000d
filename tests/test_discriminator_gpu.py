"""Discriminator (SAGAN, Ho loss) on the H100: every kernel of csrc/disc.cu through the C ABI against a float64 torch statement
of the same operation (oracle/gp_dual.py where it has one), and the whole module + adversarial criteria + WGAN-GP against the
golden fixture produced by the UNMODIFIED reference (tests/golden/discriminator.pt, oracle/make_golden.py).

Tolerances: fp32 SIMT kernels 1e-5; wgmma convolutions 3xTF32 (fp32-grade) forward / data gradient, TF32 weight gradients
(3e-3 per tensor, rel-L2)."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


@pytest.fixture(scope="module")
def L():
    from structure_knowledge_distillation_b200._cabi import lib
    return lib()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ spectral norm
@pytest.mark.parametrize("cout,cin", [(64, 19), (128, 64), (512, 256), (24, 8)])
def test_sn_power_iteration_and_weight_grad(L, cout, cin):
    from oracle import gp_dual
    g = _gen(cout + cin)
    w = torch.randn(cout, cin, 4, 4, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    u = F.normalize(torch.randn(cout, device="cuda", generator=g), dim=0)
    v = F.normalize(torch.randn(cin * 16, device="cuda", generator=g), dim=0)
    u2, v2, sigma = gp_dual.power_iteration(w.double(), u.double(), v.double())
    us, vs, sg, inv = torch.empty_like(u), torch.empty_like(v), torch.empty(1, device="cuda"), torch.empty(cout, device="cuda")
    wq = w.permute(0, 2, 3, 1)                                       # OHWI view of the same storage
    assert wq.is_contiguous()
    L.skd_sn_power_iter(cout, 16, cin, _p(wq), _p(u), _p(v), _p(us), _p(vs), _p(sg), _p(inv), cout, _st())
    assert rel(u, u2) < 1e-5 and rel(v, v2) < 1e-5 and rel(sg, sigma) < 1e-5
    assert torch.equal(us, u) and torch.equal(vs, v) and rel(inv, torch.full((cout,), 1.0 / float(sigma))) < 1e-5
    # gradient through w_bar / sigma
    cin_p = (cin + 3) // 4 * 4
    dwn = torch.randn(cout, 16, cin_p, device="cuda", generator=g)
    ref = gp_dual.sn_weight_grad(dwn[:, :, :cin].reshape(cout, 4, 4, cin).permute(0, 3, 1, 2).double(), w.double(), u2, v2, sigma)
    ws = torch.zeros(L.skd_sn_weight_grad_workspace_doubles(), device="cuda", dtype=torch.float64)
    dw = torch.zeros(cout, 4, 4, cin, device="cuda")
    for rep in range(2):                                             # second call accumulates; the workspace resets itself
        L.skd_sn_weight_grad(cout, 16, cin, cin_p, _p(dwn), _p(wq), _p(us), _p(vs), _p(sg), _p(dw), rep, _p(ws), _st())
    assert rel(dw.permute(0, 3, 1, 2), 2 * ref) < 1e-5


def test_sn_power_iteration_batched_all_layers(L):
    """skd_sn_power_iter_batched: the discriminator's four layers in one call (grid-wide phases) against float64, twice in a row
    (u, v advance in place); and bit-identical when repeated from the same state (deterministic: data-parallel replicas stay equal)."""
    import ctypes
    from oracle import gp_dual
    from structure_knowledge_distillation_b200.networks.sagan_engine import _SnLayer
    g = _gen(77)
    shapes = [(64, 19), (128, 64), (256, 128), (512, 256)]
    ws_, us_, vs_, refs = [], [], [], []
    for cout, cin in shapes:
        w = torch.randn(cout, cin, 4, 4, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        ws_.append(w)
        us_.append(F.normalize(torch.randn(cout, device="cuda", generator=g), dim=0))
        vs_.append(F.normalize(torch.randn(cin * 16, device="cuda", generator=g), dim=0))
    u0, v0 = [u.clone() for u in us_], [v.clone() for v in vs_]

    def run():
        saves = []
        descs = (_SnLayer * 4)()
        for i, (cout, cin) in enumerate(shapes):
            sv = dict(u=torch.empty(cout, device="cuda"), v=torch.empty(cin * 16, device="cuda"), sg=torch.empty(1, device="cuda"), inv=torch.empty(cout + 5, device="cuda"))
            saves.append(sv)
            descs[i] = _SnLayer(cout, 16, cin, cout + 5, _p(ws_[i].permute(0, 2, 3, 1)), _p(us_[i]), _p(vs_[i]), _p(sv["u"]), _p(sv["v"]), _p(sv["sg"]), _p(sv["inv"]))
        dp = ctypes.cast(descs, ctypes.c_void_p)
        wsp = torch.empty(L.skd_sn_power_iter_batched_workspace_floats(4, dp), device="cuda")
        L.skd_sn_power_iter_batched(4, dp, _p(wsp), _st())
        torch.cuda.synchronize()
        return saves
    first = run()
    for i, (cout, cin) in enumerate(shapes):
        u2, v2, sigma = gp_dual.power_iteration(ws_[i].double(), u0[i].double(), v0[i].double())
        assert rel(us_[i], u2) < 1e-5 and rel(vs_[i], v2) < 1e-5 and rel(first[i]["sg"], sigma) < 1e-5
        assert torch.equal(first[i]["u"], us_[i]) and torch.equal(first[i]["v"], vs_[i])
        assert rel(first[i]["inv"], torch.full((cout + 5,), 1.0 / float(sigma))) < 1e-5
        refs.append(gp_dual.power_iteration(ws_[i].double(), u2, v2))
    run()                                                            # second iteration from the advanced state
    for i in range(4):
        assert rel(us_[i], refs[i][0]) < 1e-5 and rel(vs_[i], refs[i][1]) < 1e-5
    after2 = [(u.clone(), v.clone()) for u, v in zip(us_, vs_)]
    for i in range(4):
        us_[i].copy_(u0[i]); vs_[i].copy_(v0[i])
    run(); run()
    for i in range(4):
        assert torch.equal(us_[i], after2[i][0]) and torch.equal(vs_[i], after2[i][1])


# ------------------------------------------------------------------------------------------------ BatchNorm2d(19)
@pytest.mark.parametrize("layout", ["nchw", "nhwc20"])
def test_bn2d_kernels(L, layout):
    g = _gen(7)
    B, C, H, W, Cp = 3, 19, 9, 13, 20
    if layout == "nchw":
        x = torch.randn(B, C, H, W, device="cuda", generator=g) * 2 + 0.3
    else:
        x = (torch.randn(B, H, W, Cp, device="cuda", generator=g) * 2 + 0.3).permute(0, 3, 1, 2)[:, :C]
    from structure_knowledge_distillation_b200 import ops
    xs = ops.pixel_strides(x)
    gam, bet = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    rm, rv, nbt = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"), torch.zeros((), device="cuda", dtype=torch.int64)
    ws = torch.zeros(L.skd_bn2d_workspace_doubles(), device="cuda", dtype=torch.float64)
    mean, rstd = torch.empty(32, device="cuda"), torch.empty(32, device="cuda")
    L.skd_bn2d_stats(B, C, H * W, _p(x), *xs, 1e-5, 0.1, _p(rm), _p(rv), _p(nbt), _p(mean), _p(rstd), _p(ws), _st())
    bn = torch.nn.BatchNorm2d(C).cuda().double().train()
    with torch.no_grad():
        bn.weight.copy_(gam); bn.bias.copy_(bet)
    xd = x.double().contiguous().requires_grad_(True)
    yd = bn(xd)
    assert rel(rm, bn.running_mean) < 1e-5 and rel(rv, bn.running_var) < 1e-5 and int(nbt) == 1
    out, out_lo = torch.empty(B, H, W, Cp, device="cuda"), torch.empty(B, H, W, Cp, device="cuda")
    L.skd_bn2d_apply(B, C, H * W, _p(x), *xs, _p(mean), _p(rstd), _p(gam), _p(bet), _p(out), _p(out_lo), Cp, _st())
    assert rel(out[..., :C].permute(0, 3, 1, 2), yd) < 1e-5 and float(out[..., C:].abs().max()) == 0.0
    # input gradient == symmetric Jacobian applied to dy
    dy = torch.randn(B, H, W, Cp, device="cuda", generator=g)
    (gx_ref,) = torch.autograd.grad(yd, xd, dy[..., :C].permute(0, 3, 1, 2).double(), retain_graph=True)
    sums = torch.empty(96, device="cuda")
    L.skd_bn2d_reduce(B, C, H * W, _p(x), *xs, _p(mean), _p(rstd), _p(dy), None, Cp, _p(sums), _p(ws), _st())
    dx = torch.empty_strided(x.shape, x.stride(), device="cuda")
    L.skd_bn2d_jacobian(B, C, H * W, _p(x), *xs, _p(mean), _p(rstd), _p(gam), _p(dy), Cp, _p(sums), _p(dx), *ops.pixel_strides(dx), C, None, _st())
    assert rel(dx, gx_ref) < 1e-5
    dgam, dbet = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    L.skd_bn2d_param_grad(C, B * H * W, _p(rstd), _p(sums), None, None, _p(dgam), _p(dbet), 0, _st())
    gg, gb = torch.autograd.grad(yd, [bn.weight, bn.bias], dy[..., :C].permute(0, 3, 1, 2).double())
    assert rel(dgam, gg) < 1e-5 and rel(dbet, gb) < 1e-5


# ------------------------------------------------------------------------------------------------ attention core
@pytest.mark.parametrize("tc", [1, 0])
@pytest.mark.parametrize("B,n,C,d", [(2, 128, 256, 32), (3, 32, 512, 64), (2, 35, 64, 8), (1, 6, 32, 4)])
def test_attention_forward_tangent_and_joint_backward(L, B, n, C, d, tc):
    """tc = 1: the products on the tensor cores (mma.sync m16n8k8 TF32, split precision); tc = 0: the SIMT fp32 cross-check."""
    from oracle import gp_dual
    L.skd_set_attn_tensor_cores(tc)
    try:
        _attention_case(L, B, n, C, d)
    finally:
        L.skd_set_attn_tensor_cores(1)


def _attention_case(L, B, n, C, d):
    from oracle import gp_dual
    g = _gen(n + C)
    ldq = 2 * d + C
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    qkv, tqkv = r(B * n, ldq) * 0.3, r(B * n, ldq) * 0.3
    x, tx, gy, gty = r(B * n, C), r(B * n, C), r(B * n, C), r(B * n, C)
    gamma = torch.tensor([0.37], device="cuda")
    D = lambda t: t.double().view(B, n, -1)
    q, k, v = D(qkv)[..., :d], D(qkv)[..., d:2 * d], D(qkv)[..., 2 * d:]
    tq, tk, tv = D(tqkv)[..., :d], D(tqkv)[..., d:2 * d], D(tqkv)[..., 2 * d:]
    y_ref, a_ref, o_ref = gp_dual.attn_forward(q, k, v, D(x), gamma.double())
    attn, o, y, y_lo = torch.empty(B, n, n, device="cuda"), torch.empty(B * n, C, device="cuda"), torch.empty(B * n, C, device="cuda"), torch.empty(B * n, C, device="cuda")
    L.skd_attn_fwd(B, n, C, d, _p(qkv), ldq, _p(x), _p(gamma), _p(attn), _p(o), _p(y), _p(y_lo), _st())
    assert rel(attn, a_ref) < 2e-5 and rel(o, o_ref) < 2e-5 and rel(y, y_ref) < 2e-5
    assert 0 < float(y_lo.abs().max()) <= float(y.abs().max()) * 2 ** -10        # the TF32 lo part: y - rn_tf32(y)
    ty_ref, ds_ref, da_ref, do_ref = gp_dual.attn_tangent(q, k, v, a_ref, tq, tk, tv, D(tx), gamma.double())
    dattn, to, ty = torch.empty(B, n, n, device="cuda"), torch.empty(B * n, C, device="cuda"), torch.empty(B * n, C, device="cuda")
    L.skd_attn_tangent_fwd(B, n, C, d, _p(qkv), _p(tqkv), ldq, _p(attn), _p(tx), _p(gamma), _p(dattn), _p(to), _p(ty), None, _st())
    assert rel(dattn, da_ref) < 5e-5 and rel(to, do_ref) < 5e-5 and rel(ty, ty_ref) < 5e-5
    ws = torch.empty(L.skd_attn_bwd_workspace_floats(B, n, C), device="cuda")
    # first order
    gq, gk, gv, gx, gg, *_ = gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gamma.double(), D(gy))
    gqkv, ggam = torch.empty(B * n, ldq, device="cuda"), torch.zeros(1, device="cuda")
    L.skd_attn_bwd(B, n, C, d, _p(qkv), ldq, _p(attn), _p(o), _p(gamma), _p(gy), None, None, None, None, _p(gqkv), None, _p(ggam), 0, _p(ws), _st())
    assert rel(gqkv.view(B, n, ldq), torch.cat([gq, gk, gv], -1)) < 5e-5 and rel(ggam, gg) < 5e-5
    # joint (primal, tangent)
    gq, gk, gv, gx, gg, gtq, gtk, gtv, gtx = gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gamma.double(), D(gy), tq, tk, tv, ds_ref,
                                                                         da_ref, do_ref, D(gty))
    gtqkv = torch.empty(B * n, ldq, device="cuda")
    L.skd_attn_bwd(B, n, C, d, _p(qkv), ldq, _p(attn), _p(o), _p(gamma), _p(gy), _p(tqkv), _p(dattn), _p(to), _p(gty), _p(gqkv), _p(gtqkv),
                   _p(ggam), 1, _p(ws), _st())
    assert rel(gqkv.view(B, n, ldq), torch.cat([gq, gk, gv], -1)) < 1e-4
    assert rel(gtqkv.view(B, n, ldq), torch.cat([gtq, gtk, gtv], -1)) < 1e-4
    assert rel(ggam, gg + gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gamma.double(), D(gy))[4]) < 1e-4      # accumulated onto the first-order value
    # zero primal adjoint (NULL gy): the first attention met by the penalty's reverse pass
    z = gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gamma.double(), torch.zeros_like(D(gy)), tq, tk, tv, ds_ref, da_ref, do_ref, D(gty))
    L.skd_attn_bwd(B, n, C, d, _p(qkv), ldq, _p(attn), _p(o), _p(gamma), None, _p(tqkv), _p(dattn), _p(to), _p(gty), _p(gqkv), _p(gtqkv),
                   _p(ggam), 0, _p(ws), _st())
    assert rel(gqkv.view(B, n, ldq), torch.cat(z[:3], -1)) < 1e-4 and rel(ggam, z[4]) < 1e-4


# ------------------------------------------------------------------------------------------------ convolution glue
@pytest.mark.parametrize("B,H,W,cin,cout", [(2, 65, 129, 19, 64), (2, 32, 64, 64, 128), (3, 23, 30, 64, 32), (2, 8, 16, 256, 512)])
def test_sn_conv_data_gradient_as_one_3x3_conv(L, B, H, W, cin, cout):
    """dgrad of the 4x4/s2/p1 convolution = 3x3 conv of dy into 4 parity classes (3xTF32) + un-shuffle (+ LeakyReLU mask below)."""
    g = _gen(H * W + cin)
    cin_p = (cin + 3) // 4 * 4
    w = (torch.randn(cout, cin, 4, 4, device="cuda", generator=g) * 0.1).contiguous(memory_format=torch.channels_last)
    wq = w.permute(0, 2, 3, 1)
    oh, ow = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    dy = torch.randn(B, oh, ow, cout, device="cuda", generator=g)
    ref_act = torch.randn(B, H, W, cin, device="cuda", generator=g)
    wd, wd_lo = torch.empty(4 * cin_p, 9, cout, device="cuda"), torch.empty(4 * cin_p, 9, cout, device="cuda")
    L.skd_disc_dgrad_weight_prep(cout, cin, cin_p, _p(wq), _p(wd), _p(wd_lo), _st())
    dy_lo = torch.empty_like(dy)
    L.skd_split_tf32(dy.numel(), _p(dy), None, _p(dy_lo), _st())
    hj, wj = (H + 1) // 2, (W + 1) // 2
    d2s = torch.empty(B, hj, wj, 4 * cin_p, device="cuda")
    scale = torch.full((4 * cin_p,), 0.5, device="cuda")
    L.skd_conv2d_fwd_sm100_ex(B, oh, ow, cout, 4 * cin_p, 3, 3, 1, 1, 1, _p(dy), _p(dy_lo), cout, _p(wd), _p(wd_lo), _p(d2s), 4 * cin_p, hj, wj,
                              _p(scale), None, None, 0, 0, 0.0, _st())
    out = torch.empty(B, H, W, cin_p, device="cuda")
    L.skd_disc_dgrad_unshuffle(B, H, W, cin, cin_p, _p(d2s), _p(ref_act), B, 0.1, _p(out), cin_p, None, _st())
    op = (H - ((oh - 1) * 2 - 2 + 4), W - ((ow - 1) * 2 - 2 + 4))
    ref = F.conv_transpose2d(dy.permute(0, 3, 1, 2).double(), w.double(), None, 2, 1, output_padding=op) * 0.5
    ref = ref * torch.where(ref_act.permute(0, 3, 1, 2) > 0, 1.0, 0.1)
    assert rel(out[..., :cin].permute(0, 3, 1, 2), ref) < 2e-5
    assert float(out[..., cin:].abs().max()) == 0.0 if cin_p > cin else True


@pytest.mark.parametrize("B,H,W,cin,cout,k,stride,pad,precise,res", [(8, 8, 16, 256, 512, 4, 2, 1, True, False), (8, 16, 32, 128, 256, 4, 2, 1, False, False),
                                                                     (2, 4, 8, 512, 1024, 3, 1, 1, True, False), (1, 1, 256, 640, 512, 1, 1, 0, True, True),
                                                                     (8, 32, 64, 64, 128, 4, 2, 1, True, False)])
def test_conv_split_k_matches_fp64(L, B, H, W, cin, cout, k, stride, pad, precise, res):
    """skd_conv2d_fwd_sm100_splitk: (tile, K range) work units + fixed-order partial sum + fused scale / shift / residual / leaky
    epilogue, on the discriminator's few-tile convolutions (4x8 .. 16x32 maps, K up to 4096), against float64."""
    g = _gen(H * W + cin + k)
    x = torch.randn(B, H, W, cin, device="cuda", generator=g)
    w = torch.randn(cout, k, k, cin, device="cuda", generator=g) * 0.05
    oh, ow = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    scale, shift = torch.rand(cout, device="cuda", generator=g) + 0.5, torch.randn(cout, device="cuda", generator=g)
    r = torch.randn(B, oh, ow, cout, device="cuda", generator=g) if res else None
    x_lo, w_lo = torch.empty_like(x), torch.empty_like(w)
    L.skd_split_tf32(x.numel(), _p(x), None, _p(x_lo), _st()); L.skd_split_tf32(w.numel(), _p(w), None, _p(w_lo), _st())
    nws = L.skd_conv2d_fwd_sm100_splitk_workspace_floats(B, H, W, cin, cout, k, k, stride, pad, 1, 0, 0)
    assert nws > 0, "this shape is expected to split"
    ws = torch.empty(nws, device="cuda")
    y = torch.empty(B, oh, ow, cout, device="cuda")
    L.skd_conv2d_fwd_sm100_splitk(B, H, W, cin, cout, k, k, stride, pad, 1, _p(x), _p(x_lo) if precise else None, cin, _p(w), _p(w_lo) if precise else None,
                                  _p(y), cout, 0, 0, _p(scale), _p(shift), _p(r), cout if res else 0, 1, 0.1, _p(ws), nws, _st())
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, stride, pad) * scale.double()[None, :, None, None] + shift.double()[None, :, None, None]
    if res:
        ref = ref + r.permute(0, 3, 1, 2).double()
    ref = F.leaky_relu(ref, 0.1)
    e = rel(y.permute(0, 3, 1, 2), ref)
    assert e < (5e-5 if precise else 1e-3), e            # 3xTF32, K up to 4096: the tensor-core fp32 accumulation truncates (~1e-5 per 1000 K steps)
    # and the un-split launch of the same convolution agrees (different summation order only)
    y2 = torch.empty_like(y)
    L.skd_conv2d_fwd_sm100_ex(B, H, W, cin, cout, k, k, stride, pad, 1, _p(x), _p(x_lo) if precise else None, cin, _p(w), _p(w_lo) if precise else None,
                              _p(y2), cout, 0, 0, _p(scale), _p(shift), _p(r), cout if res else 0, 1, 0.1, _st())
    assert rel(y, y2) < (5e-5 if precise else 2e-4)


def test_last_conv_adv_loss_and_gp_reductions(L):
    g = _gen(5)
    B, H, W, C = 3, 4, 8, 512
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    w = torch.randn(1, 4, 4, C, device="cuda", generator=g) * 0.05
    bias = torch.tensor([0.2], device="cuda")
    for kh, kw, hh, ww in ((4, 4, 4, 8), (2, 3, 2, 3)):
        xs = x[:, :hh, :ww].contiguous()
        oh, ow = hh - kh + 1, ww - kw + 1
        out = torch.empty(B, oh, ow, device="cuda")
        L.skd_disc_last_fwd(B, hh, ww, C, kh, kw, _p(xs), _p(w), 4 * C, _p(bias), _p(out), _st())
        xd = xs.permute(0, 3, 1, 2).double().requires_grad_(True)
        wd = w[:, :kh, :kw].permute(0, 3, 1, 2).double().requires_grad_(True)
        ref = F.conv2d(xd, wd, bias.double())
        assert rel(out, ref) < 1e-5
        gout = torch.randn(B, oh, ow, device="cuda", generator=g)
        gx_ref, gw_ref = torch.autograd.grad(ref, [xd, wd], gout.double().view(B, 1, oh, ow))
        gx = torch.empty_like(xs)
        L.skd_disc_last_dgrad(B, hh, ww, C, kh, kw, _p(gout), _p(w), 4 * C, _p(gx), None, _st())
        gw, gb = torch.zeros_like(w), torch.zeros(1, device="cuda")
        L.skd_disc_last_wgrad(B, hh, ww, C, kh, kw, _p(xs), _p(gout), _p(gw), 4 * C, _p(gb), 0, _st())
        assert rel(gx.permute(0, 3, 1, 2), gx_ref) < 1e-5 and rel(gw[:, :kh, :kw].permute(0, 3, 1, 2), gw_ref) < 1e-5
        assert rel(gb, gout.sum()) < 1e-5
    real, fake = torch.randn(40, device="cuda", generator=g), torch.randn(40, device="cuda", generator=g)
    loss, gr, gf = torch.empty((), device="cuda"), torch.empty(40, device="cuda"), torch.empty(40, device="cuda")
    for kind, fn in ((0, lambda r, f: -r.mean() + f.mean()), (1, lambda r, f: F.relu(1 - r).mean() + F.relu(1 + f).mean()), (2, lambda r, f: -f.mean())):
        rd, fd = real.double().requires_grad_(True), fake.double().requires_grad_(True)
        ref = fn(rd, fd)
        gr_ref, gf_ref = torch.autograd.grad(ref, [rd, fd], allow_unused=True)
        L.skd_adv_loss(40, _p(real), _p(fake), kind, _p(loss), _p(gr), _p(gf), _st())
        assert rel(loss, ref) < 1e-5 and rel(gf, gf_ref) < 1e-6
        if gr_ref is not None:
            assert rel(gr, gr_ref) < 1e-6
    gvec = torch.randn(4, 1000, device="cuda", generator=g) * 0.03
    norms, gpl, v = torch.empty(4, device="cuda"), torch.empty((), device="cuda"), torch.empty_like(gvec)
    L.skd_gp_norms(4, 1000, _p(gvec), 10.0, _p(norms), _p(gpl), _st())
    gd = gvec.double().requires_grad_(True)
    ref = 10.0 * ((gd.norm(dim=1) - 1) ** 2).mean()
    up = torch.tensor(0.1, device="cuda")
    L.skd_gp_direction(4, 1000, _p(gvec), _p(norms), 10.0, _p(up), _p(v), _st())
    assert rel(gpl, ref) < 1e-5 and rel(v, 0.1 * torch.autograd.grad(ref, gd)[0]) < 1e-5


# ------------------------------------------------------------------------------------------------ whole module vs the reference
def _load_from_port(D, Dp):
    sd = {k: v.clone() for k, v in Dp.state_dict().items()}
    missing = D.load_state_dict(sd, strict=True)
    return missing


def test_discriminator_wgangp_matches_reference_golden():
    """The fixture's sequence (oracle/make_golden.py::discriminator_golden): D(xs), D(xt), wgan adv loss, GP with injected alpha,
    backward.  out / attention / losses within 2e-5; spectral-norm u after three power iterations and BN running mean within 1e-5.
    Parameter gradients: per-tensor norm within 1e-2, the 16 sampled elements within 1e-1 rel-L2.  Why not tighter: the forward is
    fp32-grade (3xTF32, ~1e-5 per convolution) but not bit-identical, and LeakyReLU'(z) jumps from 0.1 to 1 at z = 0 -- one
    activation among the 32 768 of the top layer whose sign differs moves every gradient below it by 0.9 / sqrt(32768) = 5e-3
    (tools/debug_disc_chain.py shows the adjoint exact to 7e-7 up to the first mask and 4e-3 right after it; the reference's own
    stock path on this GPU, cuDNN with TF32 allowed, deviates 2e-2 from float64 by the same mechanism)."""
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.utils.criterion import CriterionAdditionalGP, CriterionAdv
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "discriminator.pt"), weights_only=False)
    torch.manual_seed(3)
    Dp = port.Discriminator(1, 19, 64)
    with torch.no_grad():
        Dp.attn1.gamma.fill_(0.3); Dp.attn2.gamma.fill_(-0.2)
    D = Discriminator(1, 19, 2, 65, 64).cuda().train()
    _load_from_port(D, Dp)
    g = cases.seeded(4)
    xs = (torch.randn(2, 19, 65, 65, generator=g) * 3).cuda()
    xt = (torch.randn(2, 19, 65, 65, generator=g) * 3).cuda()
    o_s = D(xs); o_t = D(xt)
    adv = CriterionAdv("wgan-gp")(o_s, o_t)
    crit = CriterionAdditionalGP(D, 10.0); crit.alpha = gold["alpha"].cuda()
    gp = crit([xs], [xt])
    (adv + gp).backward()
    rep = dict(out=rel(o_s[0], gold["out_s"]), p1=rel(o_s[1][:, :4, :8], gold["p1"]), adv=rel(adv, gold["adv"]), gp=rel(gp, gold["gp"]),
               u1=rel(D.l1[0].module.weight_u, gold["u1"]), bn_rm=rel(D.preprocess_additional.running_mean, gold["bn_rm"]))
    worst_n, worst_s = (0.0, None), (0.0, None)
    top = max(gd["norm"] for gd in gold["grads"].values())
    for name, p in D.named_parameters():
        gd = gold["grads"].get(name)
        # gradients that cancel analytically (e.g. attn2.value_conv.bias: d out / d (last conv input) does not depend on the input, so
        # the -mean D(T) and +mean D(S) terms cancel exactly and the penalty's tangent carries no bias) are round-off in the
        # reference's fp32 run too: compared only when they carry signal
        if gd is None or gd["norm"] < 1e-5 * top:
            continue
        mine = p.grad.detach().flatten().double().cpu()
        en = abs(float(mine.norm()) - gd["norm"]) / gd["norm"]
        es = float((mine[gd["idx"]].float() - gd["samples"]).norm() / gd["samples"].norm().clamp_min(1e-12))
        worst_n = max(worst_n, (en, name)); worst_s = max(worst_s, (es, name))
    rep["worst_grad_norm"], rep["worst_grad_samples"] = worst_n, worst_s
    print("\nPARITY discriminator_golden", rep)
    assert rep["out"] < 5e-5 and rep["p1"] < 2e-5 and rep["adv"] < 1e-4 and rep["gp"] < 1e-4     # adv = mean D(S) - mean D(T): a difference of near-equal means
    assert rep["u1"] < 1e-5 and rep["bn_rm"] < 1e-5
    assert worst_n[0] < 1e-2 and worst_s[0] < 1e-1


def _port_discriminator(H, W):
    """oracle/port.Discriminator with non-trivial attention gammas; for maps whose top level is smaller than 4x4 (46x61 logits of
    a 360x480 crop, where the reference's head cannot run) it gets the same size-aware head as ours."""
    from oracle import port
    torch.manual_seed(11)
    Dp = port.Discriminator(1, 19, 64)
    with torch.no_grad():
        Dp.attn1.gamma.fill_(-0.4); Dp.attn2.gamma.fill_(0.25)
        Dp.preprocess_additional.weight.mul_(1.2)
    return Dp


def _size_aware_head(Dp, H, W):
    hc, wc = H, W
    for _ in range(4):
        hc, wc = (hc - 2) // 2 + 1, (wc - 2) // 2 + 1
    if hc >= 4 and wc >= 4:
        return
    last = Dp.last[0]

    class _Head(torch.nn.Module):
        def forward(self, x):
            return F.conv2d(x, last.weight[:, :, :min(4, hc), :min(4, wc)], last.bias)
    Dp.last_conv = last                     # keeps the parameters registered under another name
    Dp.last = torch.nn.Sequential(_Head())


@pytest.mark.parametrize("shape,adv", [((2, 65, 129), "hinge"), ((3, 46, 61), "wgan-gp"), ((2, 65, 129), "wgan-gp")])
def test_discriminator_step_vs_port_autograd(shape, adv):
    """The step's three uses of D -- generator pass (d(-mean D(S))/d logits), then D(T), D(S), adversarial loss [+ GP], backward --
    against oracle/port.py run in float64 on the GPU with autograd (double backward for the penalty): 65x129 benchmark logits,
    and the 46x61 logits of BASELINE config 4."""
    from oracle import port
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.utils.criterion import CriterionAdditionalGP, CriterionAdv, CriterionAdvForG
    B, H, W = shape
    D = Discriminator(1, 19, B, 65, 64).cuda().train()
    _load_from_port(D, _port_discriminator(H, W))
    Dq = _port_discriminator(H, W).cuda().double().train()
    _size_aware_head(Dq, H, W)
    g = _gen(H + len(adv))
    xs = torch.randn(B, 19, H, W, device="cuda", generator=g) * 3
    xt = torch.randn(B, 19, H, W, device="cuda", generator=g) * 3
    alpha = torch.rand(B, 1, 1, 1, device="cuda", generator=g)
    xs_g = xs.clone().requires_grad_(True)
    lg = CriterionAdvForG(adv)(D(xs_g), None)
    lg.backward()
    xd = xs.double().requires_grad_(True)
    od = Dq(xd)
    lg_ref = port.adv_loss_g(od); lg_ref.backward()
    # losses are means of D outputs of both signs (|loss| can be 1e-2 of the outputs' magnitude): error measured against mean |out|;
    # gradients: LeakyReLU sign flips of single near-zero activations bound the agreement at ~5e-3 (see the golden test's docstring)
    out_scale = float(od[0].detach().abs().mean())
    assert abs(float(lg) - float(lg_ref)) < 1e-4 * out_scale and rel(xs_g.grad, xd.grad) < 1e-2
    for m in (D, Dq):
        for p in m.parameters():
            p.grad = None
    o_t, o_s = D(xt), D(xs)                                              # kd_model.py:156-157 order
    loss = CriterionAdv(adv)(o_s, o_t)
    rt, rs = Dq(xt.double()), Dq(xs.double())
    ref = port.adv_loss_d(rs, rt, adv)
    if adv == "wgan-gp":
        crit = CriterionAdditionalGP(D, 10.0); crit.alpha = alpha
        loss = loss + crit([xs], [xt])
        ref = ref + port.gradient_penalty(Dq, xs.double(), xt.double(), alpha.double(), 10.0)
    loss.backward(); ref.backward()
    assert rel(o_s[0], rs[0]) < 1e-4 and rel(o_s[2], rs[2]) < 2e-5 and abs(float(loss) - float(ref)) < 2e-4 * max(out_scale, abs(float(ref)))
    refs = dict(Dq.named_parameters())
    if hasattr(Dq, "last_conv"):
        refs["last.0.weight"], refs["last.0.bias"] = Dq.last_conv.weight, Dq.last_conv.bias
    worst = (0.0, None)
    top = max(float(q.grad.norm()) for q in refs.values() if q.grad is not None)
    for name, p in D.named_parameters():
        q = refs.get(name)
        if q is None or q.grad is None or float(q.grad.norm()) < 1e-5 * top:       # analytically cancelling gradients: round-off only
            continue
        worst = max(worst, (rel(p.grad, q.grad), name))
    print("\nPARITY discriminator_vs_port", shape, adv, "loss %.2e worst grad rel-L2 %.2e (%s)" % (rel(loss, ref), worst[0], worst[1]))
    assert worst[0] < 2e-2
