"""The pair-wise (Pa) affinity loss above 1 024 nodes against float64, element by element, with its TF32 operands pinned.

At 1 024 nodes and more `functions.PairWiseLoss` runs E = [fT^|fS^][fT^|-fS^]^T as one TF32 wgmma GEMM per image with the sum of
squares fused into the epilogue (csrc/pairwise_sm100.cu on skd_gemm_nt_sm100), and the backward as a second GEMM with E as its A
operand.  Each case runs through the C ABI on NaN-filled E, workspace, accumulator and dpooled buffers (the accumulator reused across
two calls) and once through PairWiseLoss.apply, and is held to oracle/pa_pinned.py:

  * E: every valid element within gamma_K(2^-23) sum_k |X~ W~| of the float64 product of the kernel's own TF32 operands; pad columns
    exactly 0; nothing written past the last image's rows;
  * loss: within the epilogue's derived bound (about 33 u) of sum E_got^2 / (nodes^2 N), within 1 ulp of the no-store launch, and the
    same on a second call on the same accumulator;
  * dpooled: within its pinned bound of the float64 GEMM of the kernel's own TF32(E) and Bt, through the kernel's float32 coefficient,
    and bit for bit fl(fl(coef * rS) * G) with G from skd_gemm_nt_sm100 on the same operands (the gamma_ldE bound of the GEMM is
    about 1e-3 at 8 385 nodes, as large as a wrong coefficient it must not let through);
  * dF: nonzero exactly where float64 max_pool2d's backward puts the gradient, equal there to dpooled bit for bit;
  * against true float64 (port.pairwise_loss's math per image): loss and dF within bounds derived from the TF32 unit and the data;
  * two runs give bit-identical E, dpooled and dF (the loss, a double atomic sum, within 1 ulp).

Cases: every PairWiseLoss signature at >= 1 024 nodes of one eager step of each student with the PSP level at one node per pixel, and
with the five-level list whose x1 level is at 1/65 (a guard fails on any signature INVENTORY lacks), plus synthetic rows for node
counts, channel splits, batches, windows, layouts and data the steps do not reach, and the SIMT path above 1 024 nodes.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import pa_pinned as P
from oracle import port

pytestmark = pytest.mark.gpu

NAN_BITS = 0x7FC0ABCD               # a NaN payload no kernel computes
TAIL = 67                           # NaN floats past the last row of every buffer
WORST = {}                          # check -> largest error seen as a fraction of its bound
E2E = {}                            # case -> end-to-end errors against float64


@pytest.fixture(scope="module")
def L():
    from structure_knowledge_distillation_b200._cabi import lib
    return lib()


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst error / bound per check:", {k: round(v, 4) for k, v in sorted(WORST.items())})
    print("end-to-end errors against float64:", E2E)


# ---------------------------------------------------------------------------------------------- launch signatures
def _layout_of(t):
    from structure_knowledge_distillation_b200 import ops
    sn, sc, sp = ops.pixel_strides(t)
    return ("nhwc", sp) if sc == 1 and t.shape[1] > 1 else ("nchw", 1)


def _path(nodes, cs, ct):
    from structure_knowledge_distillation_b200 import functions as Fn
    return "wgmma" if nodes >= Fn.PairWiseLoss.TCGEN05_MIN_NODES and (cs + ct) % 4 == 0 and cs % 4 == 0 else "simt"


def signature(feat_S, feat_T, ph, pw):
    """(N, nodes, C_S, C_T, H, W, ph, pw, student layout, its pixel pitch, teacher layout, its pixel pitch, path)"""
    n, cs, h, w = feat_S.shape
    ct = feat_T.shape[1]
    nodes = P.nodes_of(h, w, ph, pw)
    return (n, nodes, cs, ct, h, w, ph, pw) + _layout_of(feat_S) + _layout_of(feat_T) + (_path(nodes, cs, ct),)


def record_pairwise(monkeypatch, fn):
    """Run fn() with PairWiseLoss.apply logging the signature of every call at >= 1 024 nodes; -> the set of signatures."""
    from structure_knowledge_distillation_b200 import functions as Fn
    seen = set()
    orig = Fn.PairWiseLoss.apply

    def logged(feat_S, feat_T, ph, pw):
        sig = signature(feat_S, feat_T, ph, pw)
        if sig[1] >= Fn.PairWiseLoss.TCGEN05_MIN_NODES:
            seen.add(sig)
        return orig(feat_S, feat_T, ph, pw)
    monkeypatch.setattr(Fn.PairWiseLoss, "apply", logged)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    return seen


STUDENT_STEPS = (("resnet18", 8, 512, 1024), ("espnet_c", 16, 360, 480), ("espnet", 16, 360, 480), ("mobilenetv2", 8, 512, 1024))
RMS_E = {}


def _one_node_per_pixel(h, cap=None):
    """a pool_scale whose window is 1 x 1 on an h-row map (w < 2h): 1 / h, or `cap` (1/65) where that is smaller than 1 / h"""
    s = 1.0 / h + 1e-9
    return max(s, cap) if cap else s


def run_step(student, batch, h, w, config):
    """One eager Pa step (local Pa off): "psp" -- the scalar form on the PSP features at one node per pixel (1/65 at 512x1024);
    "levels5" -- the five-level list, x1 at 1/65 (one node per pixel where x1 has fewer than 65 rows) and the others at 0.5."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    lev = dict(lambda_pa=0.5, pool_scale=0.5) if config == "psp" else dict(lambda_pa=[0.5] * 5, pool_scale=[0.5] * 5)
    m = NetModel(make_args(batch_size=batch, pi=False, pa=True, ho=False, student=student, **lev))
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    m.forward()
    crit = m.criterion_pair_wise_for_interfeat
    if config == "psp":
        crit.scale = _one_node_per_pixel(m.preds_T[-5].shape[2])
    else:
        crit[0].scale = _one_node_per_pixel(m.preds_T[-1].shape[2], cap=1.0 / 65 + 1e-9)
    m.G_solver.zero_grad()
    m.student_backward()
    torch.cuda.synchronize()
    if config == "psp":
        RMS_E[(student, batch, h, w)] = math.sqrt(float(m.pa_G_loss))     # loss = mean of E^2 over N nodes^2
    del m
    torch.cuda.empty_cache()


# Every PairWiseLoss signature at >= 1 024 nodes of run_step for STUDENT_STEPS x ("psp", "levels5").
INVENTORY = frozenset([
    (8, 4096, 128, 512, 64, 128, 1, 2, 'nhwc', 128, 'nhwc', 512, 'wgmma'),
    (8, 8385, 128, 512, 65, 129, 1, 1, 'nhwc', 128, 'nhwc', 512, 'wgmma'),
    (8, 11008, 24, 256, 128, 256, 1, 3, 'nhwc', 24, 'nhwc', 256, 'wgmma'),
    (8, 11094, 64, 256, 129, 257, 1, 3, 'nhwc', 64, 'nhwc', 256, 'wgmma'),
    (16, 2700, 256, 512, 45, 60, 1, 1, 'nhwc', 256, 'nhwc', 512, 'wgmma'),
    (16, 7200, 19, 256, 180, 240, 2, 3, 'nhwc', 20, 'nhwc', 256, 'simt'),
])


def test_inventory_covers_every_step_signature(monkeypatch):
    seen = set()
    for st in STUDENT_STEPS:
        for config in ("psp", "levels5"):
            got = record_pairwise(monkeypatch, lambda: run_step(*st, config))
            assert got, (st, config, "no call at >= 1 024 nodes")
            seen |= got
    print("\nPA_RMS_E psp level at one node per pixel (random weights):", {k: "%.4g" % v for k, v in RMS_E.items()})
    missing = sorted(seen - INVENTORY)
    assert not missing, "signatures missing from INVENTORY:\n" + "\n".join("    %r," % (s,) for s in missing)


# ---------------------------------------------------------------------------------------------- synthetic rows
def _row(n, nodes_hw, cs, ct, win=(1, 1), lay="nhwc", data="relu", tag=""):
    h, w = nodes_hw
    sp = cs if lay != "nchw" else 1
    tl, tp = ("nhwc", ct + 2 * 512) if lay == "slice" else ((lay, ct) if lay == "nhwc" else ("nchw", 1))
    sl = "nhwc" if lay == "slice" else lay
    nodes = P.nodes_of(h, w, *win)
    return dict(sig=(n, nodes, cs, ct, h, w) + win + (sl, sp if sl == "nhwc" else 1, tl, tp, _path(nodes, cs, ct)), data=data, tag=tag)


SYNTHETIC = [
    _row(2, (32, 32), 64, 128, tag="1024 nodes: ldE = nodes, tile-aligned"),
    _row(3, (25, 41), 4, 4, lay="nchw", data="quant", tag="1025 nodes (pad 3), K = 8 under one K tile, N = 3"),
    _row(1, (65, 129), 36, 20, lay="slice", tag="8385 nodes (pad 3), concat boundary mid-tile, teacher a pitched slice"),
    _row(2, (33, 62), 4, 12, data="quant", tag="2046 nodes (pad 2), K = 16 with the concat boundary mid-tile"),
    _row(2, (65, 129), 512, 2048, win=(2, 2), data="quant", tag="K = 2560, 2x2 windows with ceil-mode edges: 2145 nodes"),
    _row(3, (65, 129), 128, 512, win=(2, 2), lay="nchw", data="quant", tag="2x2 ceil-mode, NCHW, N = 3"),
    _row(1, (25, 41), 256, 1024, tag="(256, 1024) at 1025 nodes"),
    _row(2, (32, 32), 64, 256, lay="nchw", tag="(64, 256) NCHW"),
    _row(2, (32, 33), 512, 128, tag="C_S > C_T, 1056 nodes"),
    _row(8, (46, 61), 64, 64, data="near1e-1", tag="near-teacher eps 1e-1"),
    _row(2, (46, 61), 64, 64, data="near1e-2", tag="near-teacher eps 1e-2"),
    _row(2, (46, 61), 64, 64, data="near1e-3", tag="near-teacher eps 1e-3"),
    _row(1, (129, 257), 64, 256, tag="33153 nodes: x1 at one node per pixel, E 4.4 GB"),
]

SIMT_ROWS = [_row(2, (25, 41), 19, 33), _row(1, (65, 65), 19, 33, win=(1, 1)), _row(2, (25, 41), 20, 18, lay="nchw", data="quant"),
             _row(1, (65, 65), 20, 18, data="quant")]


# ---------------------------------------------------------------------------------------------- helpers
def _st():
    return torch.cuda.current_stream().cuda_stream


def _nans(n, dtype=torch.float32):
    t = torch.empty(n, device="cuda", dtype=dtype)
    if dtype == torch.float32:
        t.view(torch.int32).fill_(NAN_BITS)
    else:
        t.fill_(float("nan"))
    return t


def _is_sentinel(t):
    return t.contiguous().view(torch.int32) == NAN_BITS


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _ulps(a, b):
    return abs(int(torch.tensor([a], dtype=torch.float32).view(torch.int32)) - int(torch.tensor([b], dtype=torch.float32).view(torch.int32)))


def _within(err, tol, check, what):
    frac = err / tol.clamp_min(1e-300)
    worst = float(frac.max()) if frac.numel() else 0.0
    WORST[check] = max(WORST.get(check, 0.0), worst)
    assert bool((err <= tol).all()), (what, check, "worst error / bound", worst)
    return worst


def _place(t, lay, pitch):
    """(N, C, H, W) float32 CUDA tensor in the given layout: NCHW, NHWC with pixel pitch `pitch` (NaN in the pad channels)"""
    if lay == "nchw":
        return t.contiguous()
    n, c, h, w = t.shape
    buf = torch.full((n, h, w, pitch), float("nan"), device="cuda")
    buf[..., :c] = t.permute(0, 2, 3, 1)
    return buf.permute(0, 3, 1, 2)[:, :c]


def _features(sig, data, seed):
    """float32-exact float64 features (N, C, H, W) on the GPU for S and T, and the student's zero-norm windows"""
    n, nodes, cs, ct, h, w, ph, pw = sig[:8]
    g = torch.Generator(device="cuda").manual_seed(seed)
    fT = torch.relu(torch.randn(n, ct, h, w, generator=g, device="cuda", dtype=torch.float64))
    zero = [(0, 0, 0), (n - 1, (h - 1) // ph, (w - 1) // pw)]          # the last one a ceil-mode edge window
    if data.startswith("near"):
        eps = float(data[4:])
        q, _ = torch.linalg.qr(torch.randn(ct, ct, generator=g, device="cuda", dtype=torch.float64))
        fS = torch.einsum("dc,ndhw->nchw", q, fT) + eps * torch.randn(n, cs, h, w, generator=g, device="cuda", dtype=torch.float64)
        zero = []
    else:
        fS = torch.relu(torch.randn(n, cs, h, w, generator=g, device="cuda", dtype=torch.float64))
        if data == "quant":
            fS = torch.round(fS * 2) / 2
    for i, y, x in zero:
        fS[i, :, y * ph:(y + 1) * ph, x * pw:(x + 1) * pw] = 0
    return fS.float().double(), fT.float().double(), zero


def _port_image(fS, fT, ph, pw):
    """port.pairwise_loss's math on one image with the window given (2x2 on 65x129 is no single pool_scale): loss and d / d fS"""
    S = fS.clone().requires_grad_(True)
    ps = F.max_pool2d(S, (ph, pw), (ph, pw), 0, ceil_mode=True)
    pt = F.max_pool2d(fT, (ph, pw), (ph, pw), 0, ceil_mode=True)
    nodes = pt.shape[2] * pt.shape[3]
    loss = ((port.affinity(pt) - port.affinity(ps)) ** 2).sum() / nodes ** 2
    (g,) = torch.autograd.grad(loss, S)
    return float(loss), g


# ---------------------------------------------------------------------------------------------- the check
def _check_wgmma(L, row, seed):
    from structure_knowledge_distillation_b200 import functions as Fn
    from structure_knowledge_distillation_b200 import ops
    sig, data = row["sig"], row["data"]
    n, nodes, cs, ct, h, w, ph, pw, sl, sp, tl, tp, path = sig
    assert path == "wgmma"
    fS, fT, zero = _features(sig, data, seed)
    S, T = _place(fS.float(), sl, sp), _place(fT.float(), tl, tp)
    pS, arg, rS = ops.pairwise_pool(S, ph, pw, True)
    pT, _, rT = ops.pairwise_pool(T, ph, pw, False)
    ldE, K, gout = ops.pad4(nodes), cs + ct, 0.75
    tot = n * nodes * ldE
    g = torch.full((), gout, device="cuda")

    # ---- forward through the C ABI: twice with E on one NaN accumulator, once with E = NULL
    ws = _nans(L.skd_pairwise_affinity_sm100_workspace_floats(n, nodes, cs, ct))
    acc = _nans(1, torch.float64)
    Es, losses = [], []
    for _ in range(2):
        E = _nans(tot + TAIL)
        loss = _nans(1)
        L.skd_pairwise_affinity_sm100(n, nodes, cs, ct, pS.data_ptr(), pT.data_ptr(), rS.data_ptr(), rT.data_ptr(), E.data_ptr(), ldE,
                                      loss.data_ptr(), ws.data_ptr(), acc.data_ptr(), _st())
        Es.append(E); losses.append(float(loss))
    loss_ns = _nans(1)
    L.skd_pairwise_affinity_sm100(n, nodes, cs, ct, pS.data_ptr(), pT.data_ptr(), rS.data_ptr(), rT.data_ptr(), None, ldE,
                                  loss_ns.data_ptr(), ws.data_ptr(), acc.data_ptr(), _st())
    torch.cuda.synchronize()
    E = Es[0]
    assert _same_bits(Es[0], Es[1]), "E differs run to run"
    del Es[1]
    assert math.isfinite(losses[0]) and _ulps(losses[0], losses[1]) <= 1, ("second call on the same accumulator", losses)
    assert _ulps(losses[0], float(loss_ns)) <= 1, ("no-store launch", losses[0], float(loss_ns))
    assert bool(_is_sentinel(E[tot:]).all()), "written past the last image's rows"
    E3 = E[:tot].view(n, nodes, ldE)
    if ldE > nodes:
        pad = E3[:, :, nodes:]
        assert bool((pad == 0).all()) and not bool(torch.signbit(pad).any()), "pad columns of E are not +0"

    # ---- backward through the C ABI: twice on NaN workspace and dpooled
    wsb = _nans(L.skd_pairwise_affinity_bwd_sm100_workspace_floats(n, nodes, cs, ldE))
    dps = []
    for _ in range(2):
        dp = _nans(n * nodes * cs + TAIL)
        L.skd_pairwise_affinity_bwd_sm100(n, nodes, cs, E.data_ptr(), ldE, pS.data_ptr(), rS.data_ptr(), g.data_ptr(), dp.data_ptr(),
                                          wsb.data_ptr(), _st())
        dps.append(dp)
    torch.cuda.synchronize()
    assert _same_bits(dps[0], dps[1]), "dpooled differs run to run"
    assert bool(_is_sentinel(dps[0][n * nodes * cs:]).all()), "dpooled written past its rows"
    dpooled = dps[0][:n * nodes * cs].view(n, nodes, cs)
    del dps, wsb, ws
    dF = torch.zeros(S.shape, device="cuda").contiguous(memory_format=torch.channels_last) if sl == "nhwc" else torch.zeros(S.shape, device="cuda")
    L.skd_pairwise_scatter(n, nodes, cs, dpooled.data_ptr(), arg.data_ptr(), dF.data_ptr(), *ops.pixel_strides(dF), _st())

    # ---- the same through PairWiseLoss.apply (its own torch.empty buffers): same bits
    Sg = S.detach().clone() if sl == "nchw" else _place(fS.float(), sl, sp)
    Sg.requires_grad_(True)
    for _ in range(2):
        lf = Fn.PairWiseLoss.apply(Sg, T, ph, pw)
        (dFa,) = torch.autograd.grad(lf, Sg, torch.full((), gout, device="cuda"))
        assert _ulps(float(lf), losses[0]) <= 1, ("PairWiseLoss.apply loss", float(lf), losses[0])
        assert _same_bits(dFa, dF), "PairWiseLoss.apply gradient differs from the C ABI's"
        del lf, dFa
    torch.cuda.empty_cache()

    # ---- dF positions: float64 max_pool2d's backward
    _, idx = F.max_pool2d(fS, (ph, pw), (ph, pw), 0, ceil_mode=True, return_indices=True)
    idx = idx.flatten(2)                                               # [N][C][nodes]
    assert torch.equal(arg.long().transpose(1, 2), idx), "arg-max is not float64 max_pool2d's"
    flat = dF.flatten(2)
    assert _same_bits(flat.gather(2, idx), dpooled.transpose(1, 2)), "dF is not dpooled at the arg-max"
    outside = torch.ones_like(flat, dtype=torch.bool).scatter_(2, idx, False)
    assert not bool((flat[outside] != 0).any()), "gradient outside the arg-max positions"

    # ---- pinned checks and float64 truth, per image in row blocks
    lrel = P.loss_rel_bound(n, nodes)
    lfe = exact = beta_terms = 0.0
    zero_rows = {(i, y * -(-w // pw) + x) for i, y, x in zero}
    frac_rest = frac_zero = 0.0
    port_loss, dF_err, dF_ref = 0.0, 0.0, 0.0
    use_port = nodes <= 12000
    for i in range(n):
        X, W = P.operands(pS[i], pT[i], rS[i], rT[i])
        Bt = P.bt_operand(pS[i], rS[i])
        cr = P.coef_rows(nodes, n, gout, rS[i])
        ex = P.exact_image(pS[i], pT[i])
        eS, eT = P.operand_rel_err(rS[i], ex["rS"]), P.operand_rel_err(rT[i], ex["rT"])
        # the backward's GEMM through the C ABI on the same operands (E, and Bt = pS * rS with zero pad columns) gives the same G
        # bits; pa_scale_kernel's product with the float32 coefficient is then pinned exactly
        Btp = torch.zeros(cs, ldE, device="cuda")
        Btp[:, :nodes] = (pS[i] * rS[i][:, None]).T
        Gk = _nans(nodes * cs).view(nodes, cs)
        L.skd_gemm_nt_sm100(nodes, cs, ldE, E3[i].data_ptr(), ldE, Btp.data_ptr(), Gk.data_ptr(), cs, None, _st())
        assert _same_bits(dpooled[i], cr[:, None] * Gk), "dpooled is not fl(fl(coef * rS) * G)"
        del Btp, Gk
        dp_true = torch.empty(nodes, cs, device="cuda", dtype=torch.float64)
        bd_true = torch.empty_like(dp_true)
        for rows in P.row_blocks(nodes, 2048 if nodes < 20000 else 1024):
            Eg = E3[i, rows, :nodes]
            Ep, BE = P.forward_block(X, W, rows)
            _within((Eg.double() - Ep).abs(), BE, "E pinned", (row["tag"], i, rows))
            del Ep, BE
            dpp, bdp = P.backward_block(Eg, Bt, cr, rows, ldE)
            err = (dpooled[i, rows].double() - dpp).abs()
            for r in range(rows.start, rows.stop):
                if (i, r) in zero_rows:
                    frac_zero = max(frac_zero, _within(err[r - rows.start], bdp[r - rows.start], "dpooled pinned, zero-norm nodes", i))
            keep = torch.ones(rows.stop - rows.start, dtype=torch.bool, device="cuda")
            for r in range(rows.start, rows.stop):
                if (i, r) in zero_rows:
                    keep[r - rows.start] = False
            frac_rest = max(frac_rest, _within(err[keep], bdp[keep], "dpooled pinned", (row["tag"], i, rows)))
            del dpp, bdp, err
            lfe += P.loss_from_rows(Eg) / nodes ** 2 / n
            Ex, beta, G, dG = P.e2e_block(ex, eS, eT, rows, nodes, n, gout, ldE)
            _within((Eg.double() - Ex).abs(), beta, "E against float64", (row["tag"], i, rows))
            exact += float(Ex.pow(2).sum()) / nodes ** 2 / n
            beta_terms += float((beta * (2 * Ex.abs() + beta)).sum()) / nodes ** 2 / n
            del Ex, beta
            dp_true[rows], bd_true[rows] = P.e2e_dpooled(G, dG, rS[i], ex["rS"], rows, nodes, n, gout)
            del G, dG
        got = flat[i].gather(1, idx[i]).T.double()                     # dF at the arg-max, [nodes][C_S]
        if use_port:                                                   # port.pairwise_loss's float64 autograd on this image
            li, gi = _port_image(fS[i:i + 1], fT[i:i + 1], ph, pw)
            port_loss += li / n
            nz, nzr = flat[i] != 0, gi[0].flatten(1) != 0
            assert torch.equal(nz, nzr), ("gradient lands elsewhere than max_pool2d's backward", i, int((nz != nzr).sum()),
                                          torch.nonzero(nz != nzr)[:4].tolist(), flat[i][nz != nzr][:4].tolist())
            ref = (gi[0].flatten(1).gather(1, idx[i]).T * (gout / n))
            assert float((ref - dp_true).abs().max()) <= 1e-9 * float(dp_true.abs().max()), "oracle float64 is not port's"
        else:
            ref = dp_true
        _within((got - ref).abs(), bd_true, "dF against float64", (row["tag"], i))
        dF_err += float((got - ref).pow(2).sum()); dF_ref += float(ref.pow(2).sum())
        torch.cuda.empty_cache()
    assert abs(losses[0] - lfe) <= lrel * lfe, ("loss against sum E^2", losses[0], lfe, lrel)
    WORST["loss vs sum E^2"] = max(WORST.get("loss vs sum E^2", 0.0), abs(losses[0] - lfe) / (lrel * lfe))
    ref_loss = port_loss if use_port else exact
    if use_port:
        assert abs(port_loss - exact) <= 1e-12 * exact
    lb = P.e2e_loss_bound(beta_terms, lrel, ref_loss)
    _within(torch.tensor(abs(losses[0] - ref_loss)), torch.tensor(lb), "loss against float64", row["tag"])
    rep = dict(loss=abs(losses[0] - ref_loss) / ref_loss, loss_bound=lb / ref_loss, dF=math.sqrt(dF_err / dF_ref),
               rms_E=math.sqrt(ref_loss), pinned_dp=frac_rest, pinned_dp_zero=frac_zero)
    E2E[row["tag"] or repr(sig)] = {k: "%.2e" % v for k, v in rep.items()}
    print("\nPARITY pa_wgmma", sig, row["data"], row["tag"], E2E[row["tag"] or repr(sig)])


def _inventory_rows():
    return [dict(sig=s, data="relu", tag="step " + repr(s)) for s in sorted(INVENTORY) if s[-1] == "wgmma"]


@pytest.mark.parametrize("row", _inventory_rows() + [r for r in SYNTHETIC if r["sig"][-1] == "wgmma"], ids=lambda r: repr(r["sig"][:8]) + r["data"])
def test_wgmma_pa_against_float64(L, row):
    _check_wgmma(L, row, seed=sum(row["sig"][:8]))
    torch.cuda.empty_cache()


def test_synthetic_rows_take_the_path_they_name():
    for r in SYNTHETIC + SIMT_ROWS:
        n, nodes, cs, ct = r["sig"][:4]
        assert r["sig"][-1] == _path(nodes, cs, ct)
    assert all(r["sig"][-1] == "wgmma" for r in SYNTHETIC) and all(r["sig"][-1] == "simt" for r in SIMT_ROWS)


# ---------------------------------------------------------------------------------------------- SIMT path above 1 024 nodes
@pytest.mark.parametrize("row", SIMT_ROWS + [dict(sig=s, data="relu", tag="step") for s in sorted(INVENTORY) if s[-1] == "simt"],
                         ids=lambda r: repr(r["sig"][:8]))
def test_simt_pa_above_1024_nodes_against_float64(row):
    """C_S = 19, or C_S + C_T not a multiple of 4: the SIMT kernels run at any node count.  Held to test_losses_gpu.py's SIMT bounds:
    loss 2e-6 relative, zero-node gradient 2e-5 rel-L2, the rest within 4x float32 torch's error plus 2e-5."""
    from structure_knowledge_distillation_b200 import functions as Fn
    n, nodes, cs, ct, h, w, ph, pw, sl, sp, tl, tp, path = row["sig"]
    fS, fT, zero = _features(row["sig"], row["data"], seed=cs * nodes)
    in_zero = torch.zeros_like(fS, dtype=torch.bool)
    for i, y, x in zero:
        in_zero[i, :, y * ph:(y + 1) * ph, x * pw:(x + 1) * pw] = True
    lref, gref = 0.0, []
    for i in range(n):
        li, gi = _port_image(fS[i:i + 1], fT[i:i + 1], ph, pw)
        lref += li / n; gref.append(gi / n)
    gref = torch.cat(gref)
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        g32 = []
        for i in range(n):
            S32 = fS[i:i + 1].float().requires_grad_(True)
            ps = F.max_pool2d(S32, (ph, pw), (ph, pw), 0, ceil_mode=True)
            pt = F.max_pool2d(fT[i:i + 1].float(), (ph, pw), (ph, pw), 0, ceil_mode=True)
            l32 = ((port.affinity(pt) - port.affinity(ps)) ** 2).sum() / nodes ** 2
            g32.append(torch.autograd.grad(l32, S32)[0].double() / n)
        g32 = torch.cat(g32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = saved

    def rel(a, b):
        return float((a - b).norm() / b.norm().clamp_min(1e-30))
    e32 = rel(g32[~in_zero], gref[~in_zero])
    runs = []
    for _ in range(2):
        S = _place(fS.float(), sl, sp).requires_grad_(True)
        loss = Fn.PairWiseLoss.apply(S, _place(fT.float(), tl, tp), ph, pw)
        (gs,) = torch.autograd.grad(loss, S)
        runs.append((loss.detach(), gs))
    assert _same_bits(runs[0][0], runs[1][0]) and _same_bits(runs[0][1], runs[1][1]), "SIMT Pa is not deterministic"
    loss, gs = runs[0]
    assert torch.equal(gs != 0, gref != 0), "gradient lands elsewhere than max_pool2d's backward"
    rep = dict(loss=abs(float(loss) - lref) / lref, grad=rel(gs.double()[~in_zero], gref[~in_zero]),
               grad_zero_nodes=rel(gs.double()[in_zero], gref[in_zero]), f32_grad=e32)
    print("\nPARITY pa_simt above 1024 nodes", row["sig"], {k: "%.2e" % v for k, v in rep.items()})
    assert rep["loss"] < 2e-6 and rep["grad_zero_nodes"] < 2e-5, rep
    assert rep["grad"] <= 4.0 * e32 + 2e-5, rep
