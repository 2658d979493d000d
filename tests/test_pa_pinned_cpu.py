"""oracle/pa_pinned.py, the float64 restatement of the wgmma pair-wise path, checked without a GPU: unrounded it is port.pairwise_loss and
its float64 autograd gradient; its TF32 rounding is test_tf32_rounding_cpu's; and its bounds hold for a float32 emulation of the kernel
(TF32 operands, float32 GEMMs, the epilogue's 32-column float32 partials) on small hand-built cases with ties and a zero-norm node."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pa_pinned as P
from oracle import port
from test_tf32_rounding_cpu import rne_tf32_bits, tf32_special_values


def _pool(f, ph, pw):
    """(N, C, H, W) float32 -> pooled rows [N][nodes][C], max_pool2d's flat indices, float32 reciprocal norms (1 / (|p| + 1e-8))"""
    p, idx = F.max_pool2d(f, (ph, pw), (ph, pw), 0, ceil_mode=True, return_indices=True)
    rows = p.flatten(2).transpose(1, 2).contiguous()
    r = (1.0 / (rows.double().pow(2).sum(2).sqrt() + 1e-8)).float()
    return rows, idx.flatten(2).transpose(1, 2), r


def _features(seed, n, c, h, w, quantize):
    g = torch.Generator().manual_seed(seed)
    f = torch.relu(torch.randn(n, c, h, w, generator=g, dtype=torch.float64))
    if quantize:
        f = torch.round(f * 2) / 2
    return f.float()


CASES = [  # n, CS, CT, h, w, ph, pw
    (2, 8, 12, 9, 11, 2, 2), (1, 4, 4, 7, 7, 1, 1), (3, 12, 20, 6, 10, 2, 3),
]


def _case(n, cs, ct, h, w, ph, pw):
    fS = _features(cs * h + w, n, cs, h, w, quantize=True)
    fT = _features(ct * h + w + 1, n, ct, h, w, quantize=False)
    fS[0, :, :ph, :pw] = 0                                            # a zero-norm student node: rS = 1e8
    fS[n - 1, :, (h - 1) // ph * ph:, (w - 1) // pw * pw:] = 0        # and the ceil-mode corner window
    return fS, fT


@pytest.mark.parametrize("n,cs,ct,h,w,ph,pw", CASES)
def test_unrounded_restatement_is_port(n, cs, ct, h, w, ph, pw):
    """Without rounding: loss and feature gradient equal port.pairwise_loss's float64 autograd (pooling windows as port chooses them)."""
    fS, fT = _case(n, cs, ct, h, w, ph, pw)
    scale = ph / h + 1e-12
    assert port.pool_patch(h, w, scale) == (ph, pw)
    Sd = fS.double().requires_grad_(True)
    ref = port.pairwise_loss(Sd, fT.double(), scale)
    (gref,) = torch.autograd.grad(ref, Sd)
    ref = ref.detach()
    pS, idx, _ = _pool(fS, ph, pw)
    pT, _, _ = _pool(fT, ph, pw)
    nodes = pS.shape[1]
    loss, grad = 0.0, torch.zeros(n, cs, h * w, dtype=torch.float64)
    g = 1.0
    for i in range(n):
        ex = P.exact_image(pS[i], pT[i])
        E = ex["X"] @ ex["W"].T
        loss += float(E.pow(2).sum()) / nodes ** 2 / n
        dp = -4.0 * g / (nodes ** 2 * n) * ex["rS"][:, None] * (E @ ex["Bt"])
        grad[i].scatter_add_(1, idx[i].T.contiguous(), dp.T.contiguous())
    assert abs(loss - float(ref)) <= 1e-13 * float(ref)
    assert torch.allclose(grad.view_as(gref), gref, rtol=1e-11, atol=1e-11 * float(gref.abs().max()))


def test_tf32_rn_is_the_hand_checked_rule():
    v = tf32_special_values()
    got = P.tf32_rn(torch.from_numpy(v.view(np.float32).copy())).numpy().view(np.uint32)
    want = rne_tf32_bits(v)
    f = v.view(np.float32)
    nan = np.isnan(f)
    assert np.array_equal(got[~nan], want[~nan]) and np.all(np.isnan(got.view(np.float32)[nan]))
    u = np.random.default_rng(3).integers(0, 2 ** 32, 100000, dtype=np.uint64).astype(np.uint32)
    u = u[~np.isnan(u.view(np.float32))]
    assert np.array_equal(P.tf32_rn(torch.from_numpy(u.view(np.float32).copy())).numpy().view(np.uint32), rne_tf32_bits(u))
    # hand-worked: ties to even down and up, a carry into the exponent, negative symmetric
    x = np.array([0x3F801000, 0x3F803000, 0x3FFFF000, 0xBF803000], dtype=np.uint32).view(np.float32)
    assert P.tf32_rn(torch.from_numpy(x.copy())).numpy().view(np.uint32).tolist() == [0x3F800000, 0x3F804000, 0x40000000, 0xBF804000]


def _emulate_kernel(pS, pT, rS, rT, N, g):
    """A float32 model of the wgmma path on the CPU: TF32 operands, float32 GEMMs, the loss as float32 partials over 32 columns added
    in double, dpooled through the same float32 coefficient."""
    nodes = pS.shape[1]
    ldE = (nodes + 3) // 4 * 4
    Es, acc = [], 0.0
    for i in range(N):
        X, W = P.operands(pS[i], pT[i], rS[i], rT[i])
        E = X.float() @ W.float().T
        Es.append(E)
        for a in range(0, nodes, P.EPI_COLS):
            part = torch.zeros(nodes, dtype=torch.float32)
            for q in range(a, min(a + P.EPI_COLS, nodes)):
                part = (part.double() + E[:, q].double() ** 2).float()     # one float32 rounding per term (an FMA)
            acc += float(part.double().sum())
    loss = float(np.float32(acc * (1.0 / (float(nodes) * nodes) / N)))
    dps = []
    for i in range(N):
        Et = P.tf32_rn(Es[i]).float()
        Bt = P.tf32_rn(pS[i] * rS[i][:, None]).float()
        G = Et @ Bt
        cr = P.coef_rows(nodes, N, g, rS[i])
        dps.append(cr[:, None] * G)
    return loss, Es, dps, ldE


@pytest.mark.parametrize("n,cs,ct,h,w,ph,pw", CASES)
def test_bounds_hold_for_a_float32_emulation(n, cs, ct, h, w, ph, pw):
    fS, fT = _case(n, cs, ct, h, w, ph, pw)
    pS, _, rS = _pool(fS, ph, pw)
    pT, _, rT = _pool(fT, ph, pw)
    assert float(rS[0, 0]) == 1e8
    nodes = pS.shape[1]
    g = 0.75
    loss, Es, dps, ldE = _emulate_kernel(pS, pT, rS, rT, n, g)
    lfe, exact_loss, beta_terms = 0.0, 0.0, 0.0
    for i in range(n):
        X, W = P.operands(pS[i], pT[i], rS[i], rT[i])
        Bt = P.bt_operand(pS[i], rS[i])
        cr = P.coef_rows(nodes, n, g, rS[i])
        ex = P.exact_image(pS[i], pT[i])
        eS, eT = P.operand_rel_err(rS[i], ex["rS"]), P.operand_rel_err(rT[i], ex["rT"])
        for rows in P.row_blocks(nodes, 5):
            Ep, BE = P.forward_block(X, W, rows)
            assert bool(((Es[i][rows].double() - Ep).abs() <= BE).all())
            dp, bd = P.backward_block(Es[i][rows], Bt, cr, rows, ldE)
            assert bool(((dps[i][rows].double() - dp).abs() <= bd).all())
            E, beta, G, dG = P.e2e_block(ex, eS, eT, rows, nodes, n, g, ldE)
            assert bool(((Es[i][rows].double() - E).abs() <= beta).all())
            dpx, bdx = P.e2e_dpooled(G, dG, rS[i], ex["rS"], rows, nodes, n, g)
            assert bool(((dps[i][rows].double() - dpx).abs() <= bdx).all())
            exact_loss += float(E.pow(2).sum()) / nodes ** 2 / n
            beta_terms += float((beta * (2 * E.abs() + beta)).sum()) / nodes ** 2 / n
        lfe += P.loss_from_rows(Es[i]) / nodes ** 2 / n
    assert abs(loss - lfe) <= P.loss_rel_bound(n, nodes) * lfe
    assert abs(loss - exact_loss) <= P.e2e_loss_bound(beta_terms, P.loss_rel_bound(n, nodes), exact_loss)


def test_bounds_are_tight_enough_to_see_a_wrong_coefficient():
    """A 1e-3 error in the backward coefficient, the size of the mutation a rel-L2 of 1e-2 would not see, leaves the pinned bound."""
    fS, fT = _case(2, 8, 12, 9, 11, 2, 2)
    pS, _, rS = _pool(fS, 2, 2)
    pT, _, rT = _pool(fT, 2, 2)
    nodes = pS.shape[1]
    _, Es, dps, ldE = _emulate_kernel(pS, pT, rS, rT, 2, 1.0)
    Bt = P.bt_operand(pS[0], rS[0])
    cr = P.coef_rows(nodes, 2, 1.0, rS[0])
    dp, bd = P.backward_block(Es[0], Bt, cr, slice(0, nodes), ldE)
    assert not bool(((dps[0].double() * 1.001 - dp).abs() <= bd).all())


def test_coefficient_rounding_is_float32():
    """coef_rows reproduces -4.f / ((float)nodes * (float)nodes * (float)N) * g * rS in float32: at 33 153 nodes nodes^2 is not a
    float32, so the float64 coefficient differs from it."""
    r = torch.tensor([1.0, 1e8, 0.37], dtype=torch.float32)
    f = np.float32
    c = f(f(-4.0) / (f(33153) * f(33153) * f(1))) * f(0.5)
    assert P.coef_rows(33153, 1, 0.5, r).tolist() == [float(f(c) * f(v)) for v in r.tolist()]
    assert float(f(c)) != -4.0 * 0.5 / 33153 ** 2
