"""Kernel-level parity on the H100 (all through the C ABI): every hand-written kernel against
  * the reference's own native kernels (libs/src/bn.cu built for sm_90a: outputs stored in tests/golden/bn_ref.pt) for the ABN ABI,
  * the CPU oracle (oracle/port.py) / the committed golden fixtures for the losses,
  * a float64 torch restatement for the convolutions (TF32 tolerance stated per test).
"""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import abn_ref, cases

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


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


# ---------------------------------------------------------------------------------------------- ABN, reference ABI
def _ref_bn():
    path = os.path.join(ROOT, "oracle", "_ref", "libbn_ref.so")
    if not os.path.exists(path):
        return None
    return ctypes.CDLL(path)


@pytest.fixture(scope="module")
def bn_gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "bn_ref.pt"), weights_only=False)


@pytest.mark.parametrize("N,C,S", abn_ref.ABN_SHAPES)
def test_bn_native_abi_matches_reference_bn_cu(L, bn_gold, N, C, S):
    """Same raw-pointer calls into our library as into the reference's bn.cu (sm_90a build; its outputs stored in
    tests/golden/bn_ref.pt, and the live library too when oracle/_ref/ holds it): <= 1e-5 relative."""
    ref = _ref_bn()
    x, w, b, dz = (t.cuda() for t in abn_ref.abn_inputs(N, C, S))
    eps = abn_ref.EPS
    mine = abn_ref.run_abi(L._dll, "skd_", N, C, S, x, w, b, dz, _st())
    # float64 restatement of bn.cu as the always-available anchor
    xd = x.double(); m = xd.mean((0, 2)); v = ((xd - m[None, :, None]) ** 2).mean((0, 2))
    assert rel(mine["mean"], m) < 1e-5 and rel(mine["var"], v) < 2e-5
    gamma = w.double().abs() + eps
    zd = (xd - m[None, :, None]) / (v + eps).sqrt()[None, :, None] * gamma[None, :, None] + b.double()[None, :, None]
    assert rel(mine["z"], zd) < 1e-5
    tol = 2e-5 if N * S >= 8 else 5e-4   # N*S == 2: dx is a difference of nearly equal numbers in both libraries
    stored = bn_gold["abn"][(N, C, S)]
    for k in mine:
        got, want = cases.at_stored(mine[k].cpu(), stored[k])
        assert rel(got, want) < tol, (k, rel(got, want))
    if ref is not None:
        theirs = abn_ref.run_abi(ref, "_", N, C, S, x, w, b, dz, _st())
        for k in mine:
            assert rel(mine[k], theirs[k]) < tol, (k, rel(mine[k], theirs[k]))


def test_activation_abi(L):
    g = torch.Generator(device="cuda").manual_seed(0)
    for n in (1, 7, 1024, 4099):
        x = torch.randn(n, device="cuda", generator=g)
        y = x.clone()
        L.skd_leaky_relu_cuda(n, y.data_ptr(), 0.01, _st())
        assert torch.equal(y, torch.where(x < 0, x * 0.01, x))
        d = torch.randn(n, device="cuda", generator=g); d0 = d.clone()
        L.skd_leaky_relu_backward_cuda(n, y.data_ptr(), d.data_ptr(), 0.01, _st())
        assert torch.equal(d, torch.where(y < 0, d0 * 0.01, d0))
        L.skd_leaky_relu_cuda(n, y.data_ptr(), 1.0 / 0.01, _st())          # inversion trick (functions.py:56-57)
        assert torch.allclose(y, x, rtol=1e-6, atol=1e-7)
        e = x.clone(); L.skd_elu_cuda(n, e.data_ptr(), _st())
        assert torch.allclose(e, F.elu(x), rtol=1e-6, atol=1e-7)
        e2 = e.clone(); L.skd_elu_inv_cuda(n, e2.data_ptr(), _st())
        assert torch.allclose(e2, x, rtol=1e-4, atol=1e-5)
        # elu backward (bn.cu:348-362): dx *= (x_out + 1) where the OUTPUT is negative -- against torch and the reference's own kernel
        d = torch.randn(n, device="cuda", generator=g); d0 = d.clone()
        L.skd_elu_backward_cuda(n, e.data_ptr(), d.data_ptr(), _st())
        assert torch.allclose(d, torch.where(e < 0, d0 * (e + 1.0), d0), rtol=1e-6, atol=1e-7)
    # elu / leaky-relu backward against the reference's own kernels: bit-exact with the stored outputs (and the live library if built)
    ref = _ref_bn()
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "bn_ref.pt"), weights_only=False)["act"]
    for n in abn_ref.ACT_SIZES:
        e, y, d = (t.cuda() for t in abn_ref.act_inputs(n))
        d_elu, d_leaky = abn_ref.run_act_backward(L._dll, "skd_", e, y, d)
        assert torch.equal(d_elu.cpu(), gold[n]["elu"]) and torch.equal(d_leaky.cpu(), gold[n]["leaky"]), n
        if ref is not None:
            r_elu, r_leaky = abn_ref.run_act_backward(ref, "_", e, y, d)
            assert torch.equal(d_elu, r_elu) and torch.equal(d_leaky, r_leaky), n


# ---------------------------------------------------------------------------------------------- ABN, fused NHWC path
@pytest.mark.parametrize("N,C,H,W,act,res,drop", [(2, 64, 9, 13, "relu", True, False), (2, 128, 7, 5, "leaky_relu", False, True),
                                                   (1, 512, 3, 3, "none", False, False), (3, 76, 5, 4, "relu", False, False),
                                                   (2, 2048, 2, 3, "leaky_relu", False, False)])
def test_abn_nhwc_fwd_bwd_vs_oracle(ops, N, C, H, W, act, res, drop):
    from oracle import port
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(N, C, H, W, generator=g) * 1.5 + 0.3
    w = torch.randn(C, generator=g); b = torch.randn(C, generator=g) * 0.2
    r = torch.randn(N, C, H, W, generator=g) if res else None
    mask = (torch.rand(N, C, generator=g) > 0.3).float() / 0.7 if drop else None
    dout = torch.randn(N, C, H, W, generator=g)
    eps, slope = 1e-5, 0.01
    # oracle (CPU, autograd through the reference-faithful ABN Function)
    xo = x.clone().requires_grad_(True); wo = w.clone().requires_grad_(True); bo = b.clone().requires_grad_(True)
    ro = r.clone().requires_grad_(True) if res else None
    rm, rv = torch.zeros(C), torch.ones(C)
    core_act = "none" if act == "relu" else act
    z = port._ABNFn.apply(xo, wo, bo, rm, rv, True, 0.1, eps, core_act, slope)
    if res: z = z + ro
    if act == "relu": z = torch.relu(z)
    if drop: z = z * mask[:, :, None, None]
    z.backward(dout)
    # ours
    dev = "cuda"
    xc = ops.to_nhwc(x.to(dev)); wc, bc = w.to(dev), b.to(dev)
    rmc, rvc = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    st = ops.abn_stats(xc, wc, bc, eps, 0.1, rmc, rvc)
    out = ops.abn_apply(xc, st[2], st[3], act, slope, residual=ops.to_nhwc(r.to(dev)) if res else None,
                        chan_mul=mask.to(dev) if drop else None)
    assert rel(out.cpu(), z.detach()) < 1e-5
    assert rel(rmc.cpu(), rm) < 1e-5 and rel(rvc.cpu(), rv) < 1e-5
    dx, dres, dw, db = ops.abn_backward(xc, out, ops.to_nhwc(dout.to(dev)), st, wc, eps, act, slope,
                                        mask.to(dev) if drop else None, res)
    assert rel(dx.cpu(), xo.grad) < 2e-4
    assert rel(dw.cpu(), wo.grad) < 2e-4 and rel(db.cpu(), bo.grad) < 2e-4
    if res:
        assert rel(dres.cpu(), ro.grad) < 1e-5
    else:
        # out = None: the activation's sign recomputed from x*scale + shift instead of read back -- bit-identical results
        dx2, _, dw2, db2 = ops.abn_backward(xc, None, ops.to_nhwc(dout.to(dev)), st, wc, eps, act, slope,
                                            mask.to(dev) if drop else None, False)
        assert torch.equal(dx2, dx) and torch.equal(dw2, dw) and torch.equal(db2, db)


# ---------------------------------------------------------------------------------------------- losses vs golden
def _golden(name):
    return torch.load(os.path.join(ROOT, "tests", "golden", name), weights_only=False)


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_losses_match_reference_goldens(ops, layout):
    """utils/criterion.py classes, run by oracle/make_golden.py on the real reference: 1e-3 relative is the contract,
    the kernels are fp32 so we hold 2e-5 on losses and 1e-4 on gradients."""
    from oracle import cases
    from structure_knowledge_distillation_b200.utils import criterion as C
    gold = _golden("criteria.pt")["criterion"]
    for name, n, cs, ct, h, w, scale, (lh, lw) in cases.CRITERION_CASES:
        S, T = cases.criterion_inputs(n, cs, ct, 19, h, w, seed=len(name) * 7 + n)
        g = cases.seeded(5 + n)
        labels = torch.randint(0, 19, (n, lh, lw), generator=g)
        labels[torch.rand(n, lh, lw, generator=g) < 0.05] = 255
        conv = (lambda t: t.cuda()) if layout == "nchw" else (lambda t: t.cuda().contiguous(memory_format=torch.channels_last))
        Sg = [conv(t).requires_grad_(True) if t is not None else None for t in S]
        Tg = [conv(t) if t is not None else None for t in T]
        pi = C.CriterionPixelWise()(Sg, Tg)
        pa = C.CriterionPairWiseforWholeFeatAfterPool(scale=scale, feat_ind=-5)(Sg, Tg)
        ce = C.CriterionDSN()(Sg, labels.cuda())
        G = gold[name]
        assert abs(float(pi) - float(G["pi"])) / abs(float(G["pi"])) < 2e-5, (name, float(pi), float(G["pi"]))
        assert abs(float(pa) - float(G["pa"])) / abs(float(G["pa"])) < 5e-5, (name, float(pa), float(G["pa"]))
        assert abs(float(ce) - float(G["ce"])) / abs(float(G["ce"])) < 2e-5, (name, float(ce), float(G["ce"]))
        (pi * 1.0 + pa * 1.0 + ce * 1.0).backward()
        assert rel(*cases.at_stored(Sg[0].grad.cpu(), cases.stored_sum(G["d_pi"], G["d_ce0"]))) < 1e-4, name
        assert rel(*cases.at_stored(Sg[1].grad.cpu(), G["d_ce1"])) < 1e-4, name
        assert rel(*cases.at_stored(Sg[2].grad.cpu(), G["d_pa"])) < 2e-4, name


@pytest.mark.parametrize("n,cs,ct,h,w", [(2, 32, 64, 33, 37), (1, 128, 512, 40, 43)])
def test_pairwise_unpooled_tcgen05_vs_oracle(ops, n, cs, ct, h, w):
    """pool window 1x1 (pool_scale -> 1/H): >= 1024 nodes -> wgmma GEMM with the L2 reduction in the epilogue; loss and
    gradient against the CPU oracle (TF32 operands: 1e-3 on the loss, 1e-2 rel-L2 on the gradient)."""
    from oracle import port
    from structure_knowledge_distillation_b200 import functions as Fn
    g = torch.Generator().manual_seed(h * w)
    fS = (torch.randn(n, cs, h, w, generator=g) + 0.5).requires_grad_(True)
    fT = torch.randn(n, ct, h, w, generator=g) + 0.5
    ref = port.pairwise_loss(fS, fT, 1.0 / min(h, w) + 1e-9)             # int(h*s) == int(w*s) == 1: 1x1 pooling window
    (gref,) = torch.autograd.grad(ref, fS)
    assert h * w >= Fn.PairWiseLoss.TCGEN05_MIN_NODES
    fSg = fS.detach().cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    loss = Fn.PairWiseLoss.apply(fSg, fT.cuda().contiguous(memory_format=torch.channels_last), 1, 1)
    loss.backward()
    assert abs(float(loss) - float(ref)) / float(ref) < 1e-3, (float(loss), float(ref))
    assert rel(fSg.grad.cpu(), gref) < 1e-2, rel(fSg.grad.cpu(), gref)
    # the SIMT path on the same inputs agrees too
    old = Fn.PairWiseLoss.TCGEN05_MIN_NODES
    Fn.PairWiseLoss.TCGEN05_MIN_NODES = 10 ** 9
    try:
        l2 = Fn.PairWiseLoss.apply(fSg.detach().requires_grad_(True), fT.cuda().contiguous(memory_format=torch.channels_last), 1, 1)
    finally:
        Fn.PairWiseLoss.TCGEN05_MIN_NODES = old
    assert abs(float(l2) - float(ref)) / float(ref) < 2e-5


def test_pairwise_affinity_full_size_north_star_shape():
    """The north-star affinity shape -- batch 8, student 128 / teacher 512 channels, 65x129 map, pool_scale 1/65 -> 8 385 nodes,
    8 385 x 8 385 x 640 per image on wgmma -- loss and gradient against oracle/port.pairwise_loss evaluated in float64 on the
    GPU (per image, to bound memory).  TF32 operands: 1e-3 on the loss, 1e-2 rel-L2 on the gradient."""
    from oracle import port
    from structure_knowledge_distillation_b200.utils.criterion import CriterionPairWiseforWholeFeatAfterPool
    g = torch.Generator(device="cuda").manual_seed(65129)
    n, cs, ct, h, w = 8, 128, 512, 65, 129
    fS = (torch.randn(n, cs, h, w, device="cuda", generator=g) + 0.5).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    fT = (torch.randn(n, ct, h, w, device="cuda", generator=g) + 0.5).contiguous(memory_format=torch.channels_last)
    crit = CriterionPairWiseforWholeFeatAfterPool(scale=1.0 / 65, feat_ind=-5)
    S = [None, None, fS, None, None, None, None]; T = [None, None, fT, None, None, None, None]
    loss = crit(S, T)
    loss.backward()
    ref_total, grads = 0.0, []
    for i in range(n):                                                     # sum over images of sum (A_T - A_S)^2 / nodes^2, then / N
        s = fS.detach()[i:i + 1].double().contiguous().requires_grad_(True)
        r = port.pairwise_loss(s, fT[i:i + 1].double().contiguous(), 1.0 / 65) / n
        (gi,) = torch.autograd.grad(r, s)
        ref_total += float(r); grads.append(gi)
    gref = torch.cat(grads)
    e_loss = abs(float(loss) - ref_total) / ref_total
    e_grad = rel(fS.grad, gref)
    print("\nPARITY pairwise_8385_nodes loss %.2e grad rel-L2 %.2e" % (e_loss, e_grad))
    assert e_loss < 1e-3 and e_grad < 1e-2


def test_pixelwise_full_size_properties(ops):
    """At BASELINE size (8,19,65,129): loss(S,S) == sum of entropies; gradient rows sum to zero; batch linearity."""
    g = torch.Generator(device="cuda").manual_seed(1)
    S = torch.randn(8, 19, 65, 129, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    T = torch.randn(8, 19, 65, 129, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    l_all = ops.pixelwise_fwd(S, T)
    l_half = ops.pixelwise_fwd(S[:4].contiguous(memory_format=torch.channels_last), T[:4].contiguous(memory_format=torch.channels_last)) + \
        ops.pixelwise_fwd(S[4:].contiguous(memory_format=torch.channels_last), T[4:].contiguous(memory_format=torch.channels_last))
    assert abs(float(l_all) - float(l_half)) / float(l_all) < 1e-6            # batch-summed, not averaged
    p = torch.softmax(S.double(), 1)
    ent = -(p * torch.log_softmax(S.double(), 1)).sum() / 65 / 129
    assert abs(float(ops.pixelwise_fwd(S, S)) - float(ent)) / float(ent) < 1e-5
    d = ops.pixelwise_bwd(S, T, torch.ones((), device="cuda"))
    assert float(d.sum(1).abs().max()) < 1e-6


# ---------------------------------------------------------------------------------------------- convolutions
def _conv_ref64(x, w, stride, pad, dil):
    return F.conv2d(x.double(), w.double(), None, stride, pad, dil)


def _tf32_trunc(t):
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


CONV_CASES = [
    (3, 64, 7, 9, 64, 3, 1, 1, 1),             # tiles that span several images (im2col wrap-around)
    (2, 32, 65, 129, 32, 3, 1, 4, 4),
    # N, Cin, H, W, Cout, k, stride, pad, dil
    (1, 32, 8, 16, 32, 1, 1, 0, 1),
    (2, 64, 9, 13, 64, 3, 1, 1, 1),
    (1, 128, 17, 19, 256, 3, 1, 2, 2),
    (1, 256, 12, 9, 512, 3, 1, 4, 4),
    (2, 64, 33, 31, 128, 3, 2, 1, 1),
    (2, 128, 33, 31, 256, 1, 2, 0, 1),
    (1, 512, 9, 9, 19, 1, 1, 0, 1),
    (1, 100, 10, 11, 72, 3, 1, 1, 1),          # channel counts that are not multiples of 32
    (2, 1024, 6, 7, 128, 3, 1, 1, 1),          # long K loop (PSP bottleneck shape class)
    (1, 64, 65, 129, 64, 3, 1, 1, 1),          # the real 1/8-resolution map with its ragged tiles
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fwd_tcgen05(ops, case):
    N, Cin, H, W, Cout, k, s, p, d = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    ref = _conv_ref64(x, w, s, p, d)
    xc = ops.to_nhwc(x); wo = ops.weight_ohwi(w)
    yd = ops.conv2d_fwd(xc, wo, s, p, d, force_direct=True)
    assert rel(yd, ref) < 1e-5, "direct SIMT conv"
    from structure_knowledge_distillation_b200._cabi import lib
    for im2col in (0, 1):                                   # rectangular tiled-mode tiles vs TMA im2col-mode tiles
        lib().skd_set_conv_im2col(im2col)
        y = ops.conv2d_fwd(xc, wo, s, p, d)
        torch.cuda.synchronize()
        assert y.shape == ref.shape
        assert rel(y, ref) < 2e-3, ("wgmma TF32 conv", im2col, rel(y, ref))          # TF32 operands, fp32 accumulate
    lib().skd_set_conv_im2col(1)


@pytest.mark.parametrize("N,Cin,H,W,Cout", [(8, 64, 9, 13, 288), (2, 128, 65, 129, 256), (3, 256, 10, 11, 1024), (2, 32, 7, 5, 160)])
def test_conv_residual_epilogue_prefetch(ops, N, Cin, H, W, Cout):
    """1x1 conv + folded BN + residual + ReLU (teacher Bottleneck conv3) in the register epilogue, incl. ragged Cout."""
    g = torch.Generator(device="cuda").manual_seed(Cout)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) / Cin ** 0.5
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5; sh = torch.randn(Cout, device="cuda", generator=g)
    res = ops.to_nhwc(torch.randn(N, Cout, H, W, device="cuda", generator=g))
    ref = torch.relu(_conv_ref64(x, w, 1, 0, 1) * sc.double()[None, :, None, None] + sh.double()[None, :, None, None] + res.double())
    out = ops.conv2d_fwd(ops.to_nhwc(x), ops.weight_ohwi(w), 1, 0, 1, scale=sc, shift=sh, residual=res, act="relu")
    assert rel(out, ref) < 2e-3, rel(out, ref)


EPILOGUE_CASES = [
    # N, Cin, H, W, Cout, k, stride, pad, dil, residual
    (1, 128, 17, 19, 256, 3, 1, 2, 2, False),      # 3 M tiles, 2 N tiles
    (2, 128, 65, 129, 256, 1, 1, 0, 1, True),      # flat GEMM with residual, 132 M tiles
    (3, 256, 10, 11, 1024, 1, 1, 0, 1, True),      # eight N tiles
    (2, 64, 33, 31, 128, 3, 2, 1, 1, False),       # stride 2
    (2, 1024, 6, 7, 136, 3, 1, 1, 1, False),       # ragged Cout: the last N tile holds 8 channels
    (1, 100, 20, 23, 72, 3, 1, 1, 1, True),        # Cout 72 -> BLOCK_N 128, 8 valid columns in the second half
    (2, 256, 65, 129, 256, 3, 1, 2, 2, False),     # teacher layer3 conv2 shape (2 images)
    (2, 64, 40, 37, 64, 3, 1, 1, 1, False),        # BLOCK_N 64 (student stem / layer1 class)
    (1, 128, 40, 37, 48, 3, 1, 1, 1, True),        # BLOCK_N 64, ragged Cout, residual
]


@pytest.mark.parametrize("case", EPILOGUE_CASES)
def test_conv_fwd_cta_pairs(ops, case):
    """The shapes that exercised Blackwell CTA pairs (multi-tile M and N, ragged Cout, stride 2, fused residual), on the wgmma kernel:
    folded-BN scale / shift (+ residual) + ReLU, im2col-mode and rectangular tiles both against the fp64 reference, and the two tile
    modes agree to TF32 summation-order noise."""
    from structure_knowledge_distillation_b200._cabi import lib
    N, Cin, H, W, Cout, k, s, p, d, with_res = case
    g = torch.Generator(device="cuda").manual_seed(sum(case[:9]))
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5; sh = torch.randn(Cout, device="cuda", generator=g)
    ref = _conv_ref64(x, w, s, p, d) * sc.double()[None, :, None, None] + sh.double()[None, :, None, None]
    res = None
    if with_res:
        res = ops.to_nhwc(torch.randn(ref.shape, device="cuda", generator=g)); ref = ref + res.double()
    ref = torch.relu(ref)
    xc = ops.to_nhwc(x); wo = ops.weight_ohwi(w)
    try:
        ys = []
        for im2col in (1, 0):
            lib().skd_set_conv_im2col(im2col)
            y = ops.conv2d_fwd(xc, wo, s, p, d, scale=sc, shift=sh, residual=res, act="relu")
            torch.cuda.synchronize()
            assert rel(y, ref) < 2e-3, ("vs fp64", im2col, rel(y, ref))
            ys.append(y)
        assert rel(ys[0], ys[1]) < 1e-3, rel(ys[0], ys[1])
    finally:
        lib().skd_set_conv_im2col(1)


@pytest.mark.parametrize("case", [(2, 64, 33, 31, 64, 3, 1, 1, 1), (1, 64, 20, 23, 128, 3, 1, 1, 1), (2, 4, 64, 67, 64, 3, 2, 1, 1),
                                  (1, 128, 17, 19, 256, 3, 1, 2, 2), (3, 64, 9, 13, 32, 1, 1, 0, 1)])
def test_conv_fwd_split_precision(ops, case):
    """3xTF32 (x_hi*w_hi + x_lo*w_hi + x_hi*w_lo per K step): fp32-grade result."""
    N, Cin, H, W, Cout, k, s, p, d = case
    g = torch.Generator(device="cuda").manual_seed(sum(case))
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    ref = _conv_ref64(x, w, s, p, d) + b.double()[None, :, None, None]
    xc = ops.to_nhwc(x).contiguous(memory_format=torch.channels_last); wo = ops.weight_ohwi(w)
    tf32 = rel(ops.conv2d_fwd(xc, wo, s, p, d, shift=b), ref)
    y = ops.conv2d_fwd_3xtf32(xc, wo, s, p, d, shift=b)
    torch.cuda.synchronize()
    assert rel(y, ref) < 2e-5, (rel(y, ref), tf32)      # tensor-core fp32 accumulation truncates: ~1e-5 (one TF32 pass: ~3e-4)
    assert tf32 > 20 * rel(y, ref)                         # the single-pass TF32 result is what the split buys us out of


def test_conv_fwd_epilogue_and_pitch(ops):
    """folded-BN scale/shift + residual + ReLU, reading a channel slice and writing into a slice of a wider buffer."""
    g = torch.Generator(device="cuda").manual_seed(7)
    N, Cin, H, W, Cout = 2, 64, 11, 14, 128
    big = torch.randn(N, H, W, 96, device="cuda", generator=g).permute(0, 3, 1, 2)
    x = big[:, 32:96]                                                       # pitch 96, offset 32
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / 24
    sc = torch.rand(Cout, device="cuda", generator=g) + 0.5; sh = torch.randn(Cout, device="cuda", generator=g)
    res = ops.to_nhwc(torch.randn(N, Cout, H, W, device="cuda", generator=g))
    obuf = torch.zeros(N, H, W, 160, device="cuda").permute(0, 3, 1, 2)
    out = obuf[:, 16:16 + Cout]
    ops.conv2d_fwd(x, ops.weight_ohwi(w), 1, 1, 1, scale=sc, shift=sh, residual=res, act="relu", out=out)
    ref = torch.relu(_conv_ref64(x, w, 1, 1, 1) * sc.double()[None, :, None, None] + sh.double()[None, :, None, None] + res.double())
    assert rel(out, ref) < 2e-3
    assert float(obuf[:, :16].abs().max()) == 0 and float(obuf[:, 16 + Cout:].abs().max()) == 0


@pytest.mark.parametrize("case", [(2, 64, 9, 13, 64, 3, 1, 1, 1), (1, 128, 17, 19, 256, 3, 1, 2, 2), (2, 64, 33, 31, 128, 3, 2, 1, 1),
                                  (2, 64, 129, 257, 128, 3, 2, 1, 1), (1, 64, 34, 32, 64, 3, 2, 1, 1),
                                  (2, 128, 33, 31, 256, 1, 2, 0, 1), (1, 256, 12, 9, 512, 3, 1, 4, 4), (1, 512, 9, 9, 128, 1, 1, 0, 1),
                                  (2, 64, 65, 129, 64, 3, 1, 1, 1)])
def test_conv_backward(ops, case):
    N, Cin, H, W, Cout, k, s, p, d = case
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 1)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).double().requires_grad_(True)
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5).double().requires_grad_(True)
    y = F.conv2d(x, w, None, s, p, d)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(dy.double())
    xc = ops.to_nhwc(x.detach().float()); dyc = ops.to_nhwc(dy); wo = ops.weight_ohwi(w.detach().float())
    dw_ref = w.grad.permute(0, 2, 3, 1)
    assert rel(ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d, force_direct=True), dw_ref) < 1e-4, "direct wgrad"
    assert rel(ops.conv2d_dgrad(dyc, wo, x.shape, s, p, d, force_direct=True), x.grad) < 1e-5, "direct dgrad"
    from structure_knowledge_distillation_b200._cabi import lib
    for linear in (0, 1):                                   # 4x8 pixel rectangles vs 32 consecutive pixels (im2col TMA) per K block
        lib().skd_set_wgrad_linear(linear)
        assert rel(ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d), dw_ref) < 2e-3, ("wgmma wgrad", linear)
    lib().skd_set_wgrad_linear(1)
    # stride 1: forward kernel on dy with flipped weights; stride 2: one stride-1 conv per input-pixel parity class
    assert rel(ops.conv2d_dgrad(dyc, wo, x.shape, s, p, d), x.grad) < 2e-3, "wgmma dgrad"


@pytest.mark.parametrize("case", [(2, 64, 33, 31, 64, False), (1, 64, 64, 72, 128, False), (2, 128, 20, 17, 64, False), (1, 64, 129, 257, 64, False),
                                  (1, 128, 65, 129, 128, False), (2, 32, 16, 8, 32, False), (1, 96, 19, 23, 100, False),
                                  (2, 64, 33, 31, 64, True), (1, 64, 40, 37, 128, True), (1, 64, 129, 257, 64, True),
                                  (2, 64, 129, 257, 128, False), (4, 128, 65, 129, 64, False), (3, 64, 129, 257, 128, True)])
def test_conv3x3_halo_kernel(ops, case):
    """The shapes of the former halo-tile kernel -- 3x3 / stride 1 / pad 1 convolutions with Cin, Cout <= 128 (the student's stem and
    layer1, their data gradients, the teacher's 64/128-wide layers) -- on the wgmma kernel through the C ABI: against float64 (TF32:
    2e-3; split precision: 2e-5), with the fused scale / shift / ReLU epilogue, ragged tiles and zero padding at the borders; the
    entry points with and without split-K workspace, and the tensor-level wrapper, agree bit for bit."""
    from structure_knowledge_distillation_b200._cabi import lib
    L = lib()
    N, Cin, H, W, Cout, precise = case
    g = torch.Generator(device="cuda").manual_seed(N + Cin + H + W + Cout)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) / (9 * Cin) ** 0.5
    scale, shift = torch.rand(Cout, device="cuda", generator=g) + 0.5, torch.randn(Cout, device="cuda", generator=g) * 0.1
    x_lo, w_lo = torch.empty_like(x), torch.empty_like(w)
    L.skd_split_tf32(x.numel(), x.data_ptr(), None, x_lo.data_ptr(), _st()); L.skd_split_tf32(w.numel(), w.data_ptr(), None, w_lo.data_ptr(), _st())
    y = torch.full((N, H, W, Cout), float("nan"), device="cuda")
    L.skd_conv2d_fwd_sm100_ex(N, H, W, Cin, Cout, 3, 3, 1, 1, 1, x.data_ptr(), x_lo.data_ptr() if precise else None, Cin, w.data_ptr(),
                              w_lo.data_ptr() if precise else None, y.data_ptr(), Cout, 0, 0, scale.data_ptr(), shift.data_ptr(), None, 0, 3,
                              0.0, _st())
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, 1, 1)
    ref = torch.relu(ref * scale.double()[None, :, None, None] + shift.double()[None, :, None, None])
    assert not torch.isnan(y).any()
    e = rel(y.permute(0, 3, 1, 2), ref)
    assert e < (2e-5 if precise else 2e-3), e
    ys = torch.full((N, H, W, Cout), float("nan"), device="cuda")
    ws = torch.empty(4, device="cuda")
    L.skd_conv2d_fwd_sm100_splitk(N, H, W, Cin, Cout, 3, 3, 1, 1, 1, x.data_ptr(), x_lo.data_ptr() if precise else None, Cin, w.data_ptr(),
                                  w_lo.data_ptr() if precise else None, ys.data_ptr(), Cout, 0, 0, scale.data_ptr(), shift.data_ptr(), None, 0,
                                  3, 0.0, ws.data_ptr(), 0, _st())
    torch.cuda.synchronize()
    assert torch.equal(ys, y)
    if not precise:
        y2 = ops.conv2d_fwd(x.permute(0, 3, 1, 2), w, 1, 1, 1, scale=scale, shift=shift, act="relu")
        assert torch.equal(y2.permute(0, 2, 3, 1), y)


@pytest.mark.parametrize("case", [(2, 512, 33, 31, 512, 3, 1, 4, 4), (1, 256, 65, 129, 256, 3, 1, 2, 2), (2, 260, 20, 17, 512, 1, 1, 0, 1),
                                  (1, 1024, 9, 11, 256, 3, 1, 1, 1), (2, 256, 33, 31, 512, 3, 2, 1, 1)])
def test_conv_wgrad_cta_pairs(ops, case):
    """The shapes that exercised Blackwell weight-gradient CTA pairs: weight gradients with several 128-wide Cout and Cin tiles (the
    teacher-sized 256 .. 1024-channel layers), both K-block modes (32 consecutive pixels through TMA im2col, pixel rectangles) within
    TF32 tolerance of float64 and close to each other."""
    from structure_knowledge_distillation_b200._cabi import lib
    N, Cin, H, W, Cout, k, s, p, d = case
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 11)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).double()
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5).double().requires_grad_(True)
    y = F.conv2d(x, w, None, s, p, d)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(dy.double())
    xc = ops.to_nhwc(x.float()); dyc = ops.to_nhwc(dy)
    dw_ref = w.grad.permute(0, 2, 3, 1)
    try:
        lib().skd_set_wgrad_linear(1)
        a = ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d)
        lib().skd_set_wgrad_linear(0)
        b = ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d)
    finally:
        lib().skd_set_wgrad_linear(1)
    assert rel(a, dw_ref) < 2e-3 and rel(b, dw_ref) < 2e-3, (rel(a, dw_ref), rel(b, dw_ref))
    assert rel(a, b) < 1e-3, rel(a, b)


@pytest.mark.parametrize("case", [(1, 256, 8, 8, 512, 4, 2, 1, 1), (2, 256, 8, 8, 512, 4, 2, 1, 1), (1, 128, 16, 16, 256, 4, 2, 1, 1),
                                  (1, 20, 65, 65, 64, 4, 2, 1, 1), (1, 512, 4, 4, 640, 1, 1, 0, 1), (3, 64, 5, 3, 32, 3, 1, 1, 1)])
def test_conv_wgrad_few_pixels(ops, case):
    """Weight gradients whose K dimension (output pixels) is smaller than one K block of the wgmma kernel (16 .. 64 pixels:
    the discriminator's top layers at batch 1-2): out-of-range pixels of the last box must contribute exact zeros."""
    N, Cin, H, W, Cout, k, s, p, d = case
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 7)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).double()
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5).double().requires_grad_(True)
    y = F.conv2d(x, w, None, s, p, d)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(dy.double())
    xc = ops.to_nhwc(x.float()); dyc = ops.to_nhwc(dy)
    dw_ref = w.grad.permute(0, 2, 3, 1)
    from structure_knowledge_distillation_b200._cabi import lib
    for linear in (0, 1):
        lib().skd_set_wgrad_linear(linear)
        try:
            e = rel(ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d), dw_ref)
        finally:
            lib().skd_set_wgrad_linear(1)
        assert e < 2e-3, ("wgmma wgrad", linear, e)


# ---------------------------------------------------------------------------------------------- pools
def test_stem_maxpool_and_psp_pyramid(ops):
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(2, 16, 22, 30, device="cuda", generator=g).requires_grad_(True)
    ref = F.max_pool2d(x, 3, 2, 1, ceil_mode=True)
    y, arg = ops.maxpool_fwd(ops.to_nhwc(x.detach()))
    assert torch.equal(y, ref)
    dy = torch.randn(ref.shape, device="cuda", generator=g)
    ref.backward(dy)
    assert rel(ops.maxpool_bwd(ops.to_nhwc(dy), arg, x.shape), x.grad) < 1e-6
    # PSP pyramid pooling + upsampling (networks/pspnet_combine.py:103,110)
    sizes = [1, 2, 3, 6]
    f = torch.randn(2, 32, 9, 13, device="cuda", generator=g).requires_grad_(True)
    pooled = ops.psp_pool_fwd(ops.to_nhwc(f.detach()), sizes)
    off = 0
    grads = torch.zeros_like(f)
    for s in sizes:
        refp = F.adaptive_avg_pool2d(f, (s, s))
        mine = pooled[:, off:off + s * s].reshape(2, s, s, 32).permute(0, 3, 1, 2)
        assert rel(mine, refp) < 1e-6
        up_ref = F.interpolate(refp, size=(9, 13), mode="bilinear", align_corners=True)
        buf = torch.zeros(2, 9, 13, 40, device="cuda").permute(0, 3, 1, 2)
        ops.psp_upsample_fwd(pooled[:, off:off + s * s].contiguous(), s, buf, 8)
        assert rel(buf[:, 8:40], up_ref) < 1e-5
        dup = torch.randn(2, 40, 9, 13, device="cuda", generator=g)
        (gp,) = torch.autograd.grad(up_ref, refp, dup[:, 8:40], retain_graph=True)
        mine_g = ops.psp_upsample_bwd(ops.to_nhwc(dup), s, 32, 8).reshape(2, s, s, 32).permute(0, 3, 1, 2)
        assert rel(mine_g, gp) < 1e-5
        off += s * s
    dpool = torch.randn(pooled.shape, device="cuda", generator=g)
    off = 0; tot = 0
    for s in sizes:
        refp = F.adaptive_avg_pool2d(f, (s, s))
        tot = tot + (refp * dpool[:, off:off + s * s].reshape(2, s, s, 32).permute(0, 3, 1, 2)).sum()
        off += s * s
    (gf,) = torch.autograd.grad(tot, f)
    assert rel(ops.psp_pool_bwd(dpool, sizes, f.shape), gf) < 1e-5


def test_sgd_step_matches_torch(ops):
    g = torch.Generator(device="cuda").manual_seed(5)
    p = torch.randn(10007, device="cuda", generator=g); p0 = p.clone()
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([ref], 0.01, momentum=0.9, weight_decay=5e-4)
    buf = torch.zeros_like(p); lr = torch.tensor(0.01, device="cuda")
    for it in range(3):
        gr = torch.randn(10007, device="cuda", generator=g)
        ref.grad = gr.clone(); opt.step()
        ops.sgd_step(p, gr, buf, lr, 0.9, 5e-4, it == 0)
    assert rel(p, ref.detach()) < 1e-6
