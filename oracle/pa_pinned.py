"""The wgmma pair-wise affinity path (csrc/pairwise_sm100.cu on skd_gemm_nt_sm100) restated in float64 with its roundings pinned, and
the error bounds of every value it produces (TEST INFRASTRUCTURE ONLY).

Inputs are the kernel's own pooled rows and reciprocal norms of ONE image, pS [nodes][C_S], pT [nodes][C_T], rS, rT [nodes] (float32,
any device); everything is computed in row blocks so that a 33 153-node image fits.

Forward.  pa_concat_norm_kernel forms X = [pT*rT | pS*rS] and W = [pT*rT | -pS*rS] as float32 products (one rounding each); the
operand tensor maps (CU_TENSOR_MAP_DATA_TYPE_TFLOAT32) round them to TF32 on load, to nearest with ties to even (`tf32_rn`, DESIGN.md
§4).  A TF32 product has 2 x 11 significant bits and is exact in float32, so the only other error is the tensor core's float32
accumulation over K = C_T + C_S products.  Model: every addition along the chain that a product passes through (within one k8 wgmma
step and across the K / 8 steps into the register accumulator) has a relative error of at most U_TC = 2^-23 of the exact partial sum
-- twice the float32 unit roundoff, so that truncation instead of round-to-nearest is covered too.  A product passes through at most K
additions, and the standard recursive-summation argument (Higham, Accuracy and Stability, Lemma 3.1 / eq. 3.5) gives

    |E_got[m][q] - E_pin[m][q]| <= gamma_K(U_TC) * sum_k |X~_mk W~_qk|,      gamma_n(u) = n u / (1 - n u),

with E_pin = X~ W~^T in float64 (X~, W~ the rounded operands).  The bound is a worst case: no tuning to any measurement.

Loss.  With E stored, conv_sm100.cu's epilogue (pass 2) squares exactly the values it stores: each thread keeps a float32 running
`fmaf(v, v, part)` over its BLOCK_N / 4 = 32 columns of one tile row (32 roundings, all terms >= 0: relative error <= gamma_32(u),
u = 2^-24), adds the partial to a double, reduces doubles across the warp and adds them atomically into one double (at most
n_part = N * nodes * ceil(nodes / 32) partials: gamma_{n_part}(2^-53)).  pa_finalize_kernel multiplies by 1 / nodes^2 / N computed in
double (2 roundings, plus 1 for the product) and rounds to float32 (u).  `loss_from_E` sums E_got^2 (exact in double) per row and then
over rows, itself within gamma_{nodes + rows}(2^-53).  Hence

    |loss - loss_from_E| <= ((1 + gamma_32(u)) (1 + gamma_{n_part}(2^-53)) (1 + gamma_{nodes + rows}(2^-53)) (1 + 3 * 2^-53) (1 + u) - 1)
                            * loss_from_E                                     (about 33 u).

Backward.  pa_transpose_norm_kernel writes Bt = pS*rS (float32 products, zero in the pad columns), the second GEMM rounds E and Bt to
TF32 and accumulates over ldE terms: G_pin = E~ Bt~^T, |G_got - G_pin| <= gamma_ldE(U_TC) * |E~| |Bt~|^T.  pa_scale_kernel then
computes dpooled = fl(fl(coef * rS_m) * G) with coef = fl(fl(-4 / fl(fl(nodes * nodes) * N)) * g) in float32 -- `coef_rows`
reproduces those float32 roundings exactly -- so with cr = fl(coef * rS_m)

    |dpooled - cr * G_pin| <= |cr| * (B_G (1 + u) + u |G_pin|).

End to end.  `exact_image` restates the same quantities without any rounding from the float32 pooled values (the norms taken in
float64), which is port.pairwise_loss in float64 (tests/test_pa_pinned_cpu.py).  `e2e_bounds` bounds the kernel against it from the
data alone: each operand element carries the TF32 rounding (2^-11), the float32 product (u) and the kernel norm's relative error rho
(measured against the float64 norm), e_m = (1 + 2^-11)(1 + u)(1 + rho_m) - 1; E then has
beta_mq = ((1 + e_m)(1 + e_q)(1 + gamma_K(U_TC)) - 1) * S_mq with S = |x| |w|^T, the loss
sum beta (2 |E| + beta) / (nodes^2 N) plus the epilogue bound, and the gradient the propagation of beta, of Bt's e and of the
TF32 rounding of E through the second GEMM and the coefficient (`e2e_bounds`).
"""
import math

import numpy as np
import torch

U = 2.0 ** -24                 # float32 unit roundoff
UD = 2.0 ** -53                # float64 unit roundoff
U_TF32 = 2.0 ** -11            # TF32 (10 explicit mantissa bits), round to nearest
U_TC = 2.0 ** -23              # tensor-core accumulation, per addition (covers truncation)
EPI_COLS = 32                  # columns of one tile row in one thread's float32 partial (BLOCK_N / 4, BLOCK_N = 128)


def gamma(n, u):
    return n * u / (1.0 - n * u)


def tf32_rn(x):
    """float32 tensor -> the nearest TF32 value (low 13 mantissa bits zero), ties to even; Inf and NaN pass (the rule of
    tests/test_tf32_rounding_cpu.py::rne_tf32_bits on torch tensors)."""
    if x.dtype != torch.float32:
        raise TypeError("tf32_rn takes float32")
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    special = (u & 0x7F800000) == 0x7F800000
    r = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    r = torch.where(special, u, r)
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32)
    return r.view(torch.float32).view(x.shape)


def _f32_products(p, r):
    """p[m][c] * r[m] as the kernels form it: one float32 rounding (exact float64 product when given float64)."""
    return p * r[:, None]


def operands(pS, pT, rS, rT, rounded=True):
    """-> (X, W) float64 [nodes][K]: the GEMM operands as the tensor core multiplies them (rounded) or unrounded."""
    xT, xS = _f32_products(pT, rT), _f32_products(pS, rS)
    X, W = torch.cat([xT, xS], 1), torch.cat([xT, -xS], 1)
    if rounded:
        X, W = tf32_rn(X), tf32_rn(W)
    return X.double(), W.double()


def row_blocks(nodes, rows=2048):
    for a in range(0, nodes, rows):
        yield slice(a, min(a + rows, nodes))


def forward_block(X, W, rows):
    """E_pin and its bound B_E on rows `rows` of one image."""
    K = X.shape[1]
    return X[rows] @ W.T, gamma(K, U_TC) * (X[rows].abs() @ W.abs().T)


def loss_rel_bound(N, nodes):
    """Relative bound of the kernel's loss against loss_from_E (see the module docstring)."""
    n_part = N * nodes * -(-nodes // EPI_COLS)
    return ((1 + gamma(EPI_COLS, U)) * (1 + gamma(n_part, UD)) * (1 + gamma(nodes + N * nodes, UD)) * (1 + 3 * UD) * (1 + U)) - 1.0


def loss_from_rows(E_rows):
    """sum of E^2 over [rows][nodes] float32 values, per row then over rows, in float64"""
    return float(E_rows.double().pow(2).sum(1).sum())


def coef_rows(nodes, N, g, rS):
    """fl(coef * rS_m) in float32, coef = fl(fl(-4 / fl(fl(nodes * nodes) * N)) * g) as pa_scale_kernel and its launch form it."""
    f = np.float32
    coef_mul = f(-4.0) / (f(nodes) * f(nodes) * f(N))
    coef = f(coef_mul) * f(g)
    return torch.tensor(float(coef), dtype=torch.float32, device=rS.device) * rS


def bt_operand(pS, rS):
    """Bt~ as [nodes][C_S] float64 (transposed back): TF32 of the float32 products pS * rS"""
    return tf32_rn(_f32_products(pS, rS)).double()


def backward_block(E_rows, Bt, cr, rows, ldE):
    """From the kernel's own stored E rows [rows][nodes] (float32): dpooled_pin and its elementwise bound on rows `rows`."""
    Et = tf32_rn(E_rows.contiguous()).double()
    G = Et @ Bt
    BG = gamma(ldE, U_TC) * (Et.abs() @ Bt.abs())
    c = cr[rows].double()[:, None]
    return c * G, c.abs() * (BG * (1 + U) + U * G.abs())


# ---------------------------------------------------------------------------------------------- float64 truth and the end-to-end bound
def exact_norms(p):
    """float64 reciprocal norms of float32 pooled rows: 1 / (|p| + 1e-8) (utils.py's eps outside the sqrt)"""
    return 1.0 / (p.double().pow(2).sum(1).sqrt() + 1e-8)


def exact_image(pS, pT):
    """-> dict of the unrounded float64 quantities of one image: x / w operands, Bt, the norms."""
    rS, rT = exact_norms(pS), exact_norms(pT)
    pSd, pTd = pS.double(), pT.double()
    X, W = operands(pSd, pTd, rS, rT, rounded=False)
    return dict(X=X, W=W, Bt=pSd * rS[:, None], rS=rS, rT=rT)


def operand_rel_err(r_kernel, r_exact):
    """e_m of each node's operand row: TF32 rounding, the float32 product and the kernel norm's measured relative error."""
    rho = (r_kernel.double() / r_exact - 1.0).abs()
    return (1 + U_TF32) * (1 + U) * (1 + rho) - 1.0


def e2e_block(ex, eS, eT, rows, nodes, N, g, ldE):
    """Rows `rows` of one image: (E, bound on |E_kernel - E|, G, bound on |G_kernel - G| (before the coefficient)).  eS / eT: per-node
    operand errors (operand_rel_err) of the student and teacher halves."""
    X, W, Bt = ex["X"], ex["W"], ex["Bt"]
    K = X.shape[1]
    e = torch.maximum(eS, eT)
    E = X[rows] @ W.T
    S = X[rows].abs() @ W.abs().T
    gk = gamma(K, U_TC)
    beta = ((1 + e[rows])[:, None] * (1 + e)[None, :] * (1 + gk) - 1.0) * S
    betap = beta + U_TF32 * (E.abs() + beta)                    # the TF32 rounding of E as the backward GEMM's operand
    gl = gamma(ldE, U_TC)
    emax = float(eS.max())
    G = E @ Bt
    dG = (betap * (1 + emax) * (1 + gl) + E.abs() * (emax + gl * (1 + emax))) @ Bt.abs()
    return E, beta, G, dG


def e2e_dpooled(G, dG, rS_kernel, rS_exact, rows, nodes, N, g):
    """dpooled in float64 (-4 g / (nodes^2 N) r_m G) and the kernel's bound: the coefficient's float32 roundings (6 u, with its
    two products), the kernel norm's relative error rho_m, and dG."""
    c = -4.0 * g / (float(nodes) ** 2 * N) * rS_exact[rows][:, None]
    rho = (rS_kernel[rows].double() / rS_exact[rows] - 1.0).abs()[:, None]
    eta = (1 + U) ** 6 * (1 + rho) - 1.0
    return c * G, c.abs() * (eta * G.abs() + (1 + eta) * dG)


def e2e_loss_bound(sum_beta_terms, loss_kernel_rel, loss_exact):
    """|loss_kernel - loss| <= sum beta (2 |E| + beta) / (nodes^2 N) (accumulated by the caller, already divided) plus the
    epilogue's relative bound on the kernel's own E."""
    return sum_beta_terms + loss_kernel_rel * (loss_exact + sum_beta_terms)


def nodes_of(h, w, ph, pw):
    return math.ceil(h / ph) * math.ceil(w / pw)
