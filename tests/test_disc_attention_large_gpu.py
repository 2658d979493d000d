"""The discriminator's self-attention beyond 128 positions (the row-stripe kernels of csrc/disc.cu) on the H100.

Crops larger than 512x1024 put more than 128 positions under attn1 (769x769: 144, 1024x1024: 256, 1024x2048: 512).  Checked here:
the forward, tangent and the three backward modes against oracle/gp_dual.py in float64 (the tolerances of the n <= 128 kernels'
test), the forced row-stripe path against the whole-tile kernels at n = 128, the bound, determinism, and the whole discriminator
(generator pass, D(T), D(S), adversarial loss [+ GP], backward) against oracle/port.py in float64 at the logit sizes of those crops."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_N = 1024


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


class _Mode:
    """skd_set_attn_tensor_cores / skd_set_attn_tiled for the duration of a block, restored to the defaults after it."""

    def __init__(self, L, tc=1, tiled=0):
        self.L, self.tc, self.tiled = L, tc, tiled

    def __enter__(self):
        self.L.skd_set_attn_tensor_cores(self.tc); self.L.skd_set_attn_tiled(self.tiled)

    def __exit__(self, *exc):
        self.L.skd_set_attn_tensor_cores(1); self.L.skd_set_attn_tiled(0)


def _inputs(B, n, C, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ldq = 2 * d + C
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    return dict(B=B, n=n, C=C, d=d, ldq=ldq, qkv=r(B * n, ldq) * 0.3, tqkv=r(B * n, ldq) * 0.3, x=r(B * n, C), tx=r(B * n, C),
                gy=r(B * n, C), gty=r(B * n, C), gamma=torch.tensor([0.37], device="cuda"))


def _run_all(L, I):
    """Every entry point once, in the order the discriminator uses them: forward, tangent, first-order, joint and NULL-gy backward."""
    B, n, C, d, ldq = I["B"], I["n"], I["C"], I["d"], I["ldq"]
    e = lambda *s: torch.empty(*s, device="cuda")
    out = dict(attn=e(B, n, n), o=e(B * n, C), y=e(B * n, C), y_lo=e(B * n, C), dattn=e(B, n, n), to=e(B * n, C), ty=e(B * n, C))
    L.skd_attn_fwd(B, n, C, d, _p(I["qkv"]), ldq, _p(I["x"]), _p(I["gamma"]), _p(out["attn"]), _p(out["o"]), _p(out["y"]), _p(out["y_lo"]), _st())
    L.skd_attn_tangent_fwd(B, n, C, d, _p(I["qkv"]), _p(I["tqkv"]), ldq, _p(out["attn"]), _p(I["tx"]), _p(I["gamma"]), _p(out["dattn"]),
                           _p(out["to"]), _p(out["ty"]), None, _st())
    ws = torch.full((L.skd_attn_bwd_workspace_floats(B, n, C),), float("nan"), device="cuda")      # every read element must be written first
    out["g1"], out["gg1"] = e(B * n, ldq), torch.zeros(1, device="cuda")
    L.skd_attn_bwd(B, n, C, d, _p(I["qkv"]), ldq, _p(out["attn"]), _p(out["o"]), _p(I["gamma"]), _p(I["gy"]), None, None, None, None,
                   _p(out["g1"]), None, _p(out["gg1"]), 0, _p(ws), _st())
    out["g2"], out["gt2"], out["gg2"] = e(B * n, ldq), e(B * n, ldq), out["gg1"].clone()
    L.skd_attn_bwd(B, n, C, d, _p(I["qkv"]), ldq, _p(out["attn"]), _p(out["o"]), _p(I["gamma"]), _p(I["gy"]), _p(I["tqkv"]), _p(out["dattn"]),
                   _p(out["to"]), _p(I["gty"]), _p(out["g2"]), _p(out["gt2"]), _p(out["gg2"]), 1, _p(ws), _st())
    out["g3"], out["gt3"], out["gg3"] = e(B * n, ldq), e(B * n, ldq), torch.zeros(1, device="cuda")
    L.skd_attn_bwd(B, n, C, d, _p(I["qkv"]), ldq, _p(out["attn"]), _p(out["o"]), _p(I["gamma"]), None, _p(I["tqkv"]), _p(out["dattn"]),
                   _p(out["to"]), _p(I["gty"]), _p(out["g3"]), _p(out["gt3"]), _p(out["gg3"]), 0, _p(ws), _st())
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("tc", [1, 0])
@pytest.mark.parametrize("B,n,C,d", [(2, 144, 256, 32), (1, 256, 256, 32), (1, 512, 256, 32), (2, 129, 512, 64), (1, 200, 64, 8),
                                     (1, MAX_N, 256, 32), (1, MAX_N, 512, 64), (2, 128, 512, 64)])
def test_large_attention_matches_float64(L, B, n, C, d, tc):
    """tc = 1: products on mma.sync TF32 in split precision; tc = 0: the SIMT fp32 cross-check.  (2, 128, 512, 64) is attn2 of a
    1024x2048 crop: its whole-tile tangent and joint backward would need 259 KB of shared memory, so they run as row stripes."""
    from oracle import gp_dual
    I = _inputs(B, n, C, d, n + C)
    with _Mode(L, tc=tc):
        out = _run_all(L, I)
    D = lambda t: t.double().view(B, n, -1)
    q, k, v = D(I["qkv"])[..., :d], D(I["qkv"])[..., d:2 * d], D(I["qkv"])[..., 2 * d:]
    tq, tk, tv = D(I["tqkv"])[..., :d], D(I["tqkv"])[..., d:2 * d], D(I["tqkv"])[..., 2 * d:]
    gm = I["gamma"].double()
    y_ref, a_ref, o_ref = gp_dual.attn_forward(q, k, v, D(I["x"]), gm)
    assert rel(out["attn"], a_ref) < 2e-5 and rel(out["o"], o_ref) < 2e-5 and rel(out["y"], y_ref) < 2e-5
    assert 0 < float(out["y_lo"].abs().max()) <= float(out["y"].abs().max()) * 2 ** -10
    ty_ref, ds_ref, da_ref, do_ref = gp_dual.attn_tangent(q, k, v, a_ref, tq, tk, tv, D(I["tx"]), gm)
    assert rel(out["dattn"], da_ref) < 5e-5 and rel(out["to"], do_ref) < 5e-5 and rel(out["ty"], ty_ref) < 5e-5
    first = gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gm, D(I["gy"]))
    assert rel(out["g1"].view(B, n, -1), torch.cat(first[:3], -1)) < 5e-5 and rel(out["gg1"], first[4]) < 5e-5
    joint = gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gm, D(I["gy"]), tq, tk, tv, ds_ref, da_ref, do_ref, D(I["gty"]))
    assert rel(out["g2"].view(B, n, -1), torch.cat(joint[:3], -1)) < 1e-4
    assert rel(out["gt2"].view(B, n, -1), torch.cat(joint[5:8], -1)) < 1e-4
    assert rel(out["gg2"], joint[4] + first[4]) < 1e-4                          # accumulated onto the first-order value
    z = gp_dual.attn_joint_backward(q, k, v, a_ref, o_ref, gm, torch.zeros_like(D(I["gy"])), tq, tk, tv, ds_ref, da_ref, do_ref, D(I["gty"]))
    assert rel(out["g3"].view(B, n, -1), torch.cat(z[:3], -1)) < 1e-4
    assert rel(out["gt3"].view(B, n, -1), torch.cat(z[5:8], -1)) < 1e-4 and rel(out["gg3"], z[4]) < 1e-4


@pytest.mark.parametrize("tc", [1, 0])
@pytest.mark.parametrize("B,n,C,d", [(2, 128, 256, 32), (2, 128, 512, 64), (3, 100, 512, 64)])
def test_row_stripe_kernels_agree_with_whole_tile_kernels(L, B, n, C, d, tc):
    """skd_set_attn_tiled(1) sends n <= 128 through the row-stripe kernels: every output within 2e-5 of the whole-tile kernels (the
    ones whose tiles fit shared memory: at (n, d) = (128, 64) the tangent and joint backward are row stripes either way)."""
    I = _inputs(B, n, C, d, 7 + C)
    with _Mode(L, tc=tc, tiled=0):
        old = _run_all(L, I)
    with _Mode(L, tc=tc, tiled=1):
        new = _run_all(L, I)
    for key in ("attn", "o", "y", "dattn", "to", "ty", "g1", "gg1", "g2", "gt2", "gg2", "g3", "gt3", "gg3"):
        assert rel(new[key], old[key]) < 2e-5, key


def test_workspace_covers_the_dispatched_path(L):
    """The row-stripe backward needs 2 B n^2 + B n floats whatever C is; the whole-tile backward B (C / 32) 2 n^2 + B C / 32.  For
    n <= 128 either may run, so the larger is returned (unchanged for C > 32)."""
    assert L.skd_attn_bwd_workspace_floats(8, 128, 256) == 8 * 8 * 2 * 128 * 128 + 8 * 8
    assert L.skd_attn_bwd_workspace_floats(8, 128, 32) == 2 * 8 * 128 * 128 + 8 * 128
    assert L.skd_attn_bwd_workspace_floats(8, 512, 256) == 2 * 8 * 512 * 512 + 8 * 512
    assert L.skd_attn_bwd_workspace_floats(1, MAX_N, 512) == 2 * MAX_N * MAX_N + MAX_N


def test_one_past_the_bound_raises(L):
    n, C, d, B = MAX_N + 1, 256, 32, 1
    ldq = 2 * d + C
    buf = torch.zeros(B * n * max(ldq, n), device="cuda")
    g = torch.ones(1, device="cuda")
    with pytest.raises(RuntimeError, match="skd_attn_fwd.*1024"):
        L.skd_attn_fwd(B, n, C, d, _p(buf), ldq, _p(buf), _p(g), _p(buf), _p(buf), _p(buf), None, _st())
    with pytest.raises(RuntimeError, match="skd_attn_tangent_fwd.*1024"):
        L.skd_attn_tangent_fwd(B, n, C, d, _p(buf), _p(buf), ldq, _p(buf), _p(buf), _p(g), _p(buf), _p(buf), _p(buf), None, _st())
    with pytest.raises(RuntimeError, match="skd_attn_bwd.*1024"):
        L.skd_attn_bwd(B, n, C, d, _p(buf), ldq, _p(buf), _p(buf), _p(g), _p(buf), None, None, None, None, _p(buf), None, _p(g), 0, _p(buf), _st())


@pytest.mark.parametrize("n", [144, 512])
def test_row_stripe_kernels_are_deterministic(L, n):
    """Fixed-order sums, no atomics: two identical calls of every entry point give bit-identical outputs."""
    I = _inputs(4, n, 256, 32, 3)
    a, b = _run_all(L, I), _run_all(L, I)
    for key in a:
        assert torch.equal(a[key], b[key]), key


# ------------------------------------------------------------------------------------------------ whole discriminator
def _port_discriminator():
    from oracle import port
    torch.manual_seed(11)
    Dp = port.Discriminator(1, 19, 64)
    with torch.no_grad():
        Dp.attn1.gamma.fill_(-0.4); Dp.attn2.gamma.fill_(0.25)
        Dp.preprocess_additional.weight.mul_(1.2)
    return Dp


@pytest.mark.parametrize("shape,adv", [((2, 97, 97), "wgan-gp"), ((1, 129, 129), "hinge"), ((1, 129, 257), "wgan-gp")])
def test_discriminator_step_vs_port_at_large_crops(shape, adv):
    """Logits of 769x769 (attn1 over 144 positions), 1024x1024 (256) and 1024x2048 (512) crops: the generator pass, then D(T), D(S),
    adversarial loss [+ GP], backward, against oracle/port.py in float64 with autograd (double backward for the penalty)."""
    from oracle import port
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.utils.criterion import CriterionAdditionalGP, CriterionAdv, CriterionAdvForG
    B, H, W = shape
    D = Discriminator(1, 19, B, 65, 64).cuda().train()
    D.load_state_dict({k: v.clone() for k, v in _port_discriminator().state_dict().items()}, strict=True)
    Dq = _port_discriminator().cuda().double().train()
    g = torch.Generator(device="cuda").manual_seed(H + W + len(adv))
    xs = torch.randn(B, 19, H, W, device="cuda", generator=g) * 3
    xt = torch.randn(B, 19, H, W, device="cuda", generator=g) * 3
    alpha = torch.rand(B, 1, 1, 1, device="cuda", generator=g)
    xs_g = xs.clone().requires_grad_(True)
    lg = CriterionAdvForG(adv)(D(xs_g), None)
    lg.backward()
    xd = xs.double().requires_grad_(True)
    od = Dq(xd)
    lg_ref = port.adv_loss_g(od); lg_ref.backward()
    out_scale = float(od[0].detach().abs().mean())
    assert abs(float(lg) - float(lg_ref)) < 1e-4 * out_scale and rel(xs_g.grad, xd.grad) < 1e-2
    for m in (D, Dq):
        for p in m.parameters():
            p.grad = None
    o_t, o_s = D(xt), D(xs)                                              # kd_model.py:156-157 order
    loss = CriterionAdv(adv)(o_s, o_t)
    rt, rs = Dq(xt.double()), Dq(xs.double())
    h3, w3 = H, W
    for _ in range(3):
        h3, w3 = (h3 - 2) // 2 + 1, (w3 - 2) // 2 + 1
    assert tuple(o_s[1].shape) == (B, h3 * w3, h3 * w3) and h3 * w3 > 128 and rel(o_s[1], rs[1]) < 2e-5
    ref = port.adv_loss_d(rs, rt, adv)
    if adv == "wgan-gp":
        crit = CriterionAdditionalGP(D, 10.0); crit.alpha = alpha
        loss = loss + crit([xs], [xt])
        ref = ref + port.gradient_penalty(Dq, xs.double(), xt.double(), alpha.double(), 10.0)
    loss.backward(); ref.backward()
    assert rel(o_s[0], rs[0]) < 1e-4 and rel(o_s[2], rs[2]) < 2e-5 and abs(float(loss) - float(ref)) < 2e-4 * max(out_scale, abs(float(ref)))
    refs = dict(Dq.named_parameters())
    worst = (0.0, None)
    top = max(float(q.grad.norm()) for q in refs.values() if q.grad is not None)
    for name, p in D.named_parameters():
        q = refs.get(name)
        if q is None or q.grad is None or float(q.grad.norm()) < 1e-5 * top:       # analytically cancelling gradients: round-off only
            continue
        worst = max(worst, (rel(p.grad, q.grad), name))
    print("\nPARITY discriminator_vs_port", shape, adv, "attn1 n = %d" % rs[1].shape[1],
          "loss %.2e worst grad rel-L2 %.2e (%s)" % (rel(loss, ref), worst[0], worst[1]))
    assert worst[0] < 2e-2
