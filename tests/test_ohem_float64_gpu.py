"""The OHEM cross entropy (OhemCrossEntropy2d / CriterionOhemDSN) against float64 over the class counts, zoom factors, layouts and grid
geometries where its three pieces can go wrong: the 1/factor grid of p[label] (csrc/ohem.cu ohem_grid_kernel), the radix select of the
order statistic (ohem_hist / ohem_select), and the masked cross entropy with its gradients (the OHEM row kernel, ohem_finalize_kernel and
skd_ohem_dsn_ce_bwd_cols of csrc/losses.cu).

The float64 reference runs on the GPU: the align_corners upsample and the softmax in float64, then scipy's zoom (order 1 for the
probabilities, order 0 for the labels) restated in torch by tools/ohem_oracle.ohem_grid64, which test_ohem_float64_cpu.py pins bit for bit
against scipy.ndimage.zoom.  The masked loss is compared with w0 * CE(up0)[p64 <= thr] + w1 * CE(up1) at the kernel's own float32 threshold;
pixels whose float64 probability lies too close to the threshold to decide are set to ignore first, unless they are the source of a grid
label.  Where a grid point lies exactly on a pixel its value IS that pixel's probability, and the reference keeps the pixel that defines
the threshold (p <= p): the kept counts are checked as exact integers there.  Peaked (randn x 20) and offset (+1e3) logits use the same
reference in float32 torch as the yardstick.  Every case runs twice and must give bit-identical results.

Bounds, against the worst error measured on an H100 80GB HBM3 (700 W power limit), printed per test on a PARITY line: grid values 2e-4
(measured 4.4e-5, the float32 source coordinate at 512 x 1024); masked loss 2e-6, gradient 2e-5 and edge 2e-5, the bounds of
test_losses_gpu.py (measured 1.0e-7, 3.0e-6 and 4.3e-6); peaked and offset logits within 4x float32 torch's error plus a floor (the kernel
measured at 0.9-1.3x float32 torch on the grid).  Kept counts, valid counts, grid labels and thresholds are exact."""
import pytest
import torch
import torch.nn.functional as F

from tools import ohem_oracle as O

pytestmark = pytest.mark.gpu

CLASSES = [1, 2, 3, 4, 7, 19, 20, 21, 31, 32]
LAYOUTS = ("nchw", "nhwc", "pad4")
# grid values, relative, unit-scale logits: the kernel's source coordinate (h - 1) / (H - 1) * Y is float32, as ATen's, so p[label]
# follows float32 torch at the full-resolution pixels, up to ~4e-5 from float64 at the benchmark's 65 x 129 -> 512 x 1024
GRID_TOL = 2e-4
LOSS_TOL = 2e-6            # relative, losses against float64
GRAD_TOL = 2e-5            # rel-L2, gradients against float64
EDGE_TOL = 2e-5            # worst element on the first / last logit row and column, relative to the largest gradient element
F32_FACTOR = 4.0           # peaked and offset logits: up to 4x float32 torch's error plus a floor
PEAK_GRID_FLOOR = 1e-5
PEAK_LOSS_FLOOR = 1e-5
PEAK_GRAD_FLOOR = 1e-4
# relative distance to the threshold inside which a pixel's keep decision is left to float32 rounding: a few times the float32 error
# of p[label] for each kind of logits (the offset logits carry ~1e-4 of it from their 1e3 magnitude alone)
UNDECIDED = dict(randn=1e-5, peaked=1e-4, offset=1e-3)

# (h, w), (H, W), factor; (h, w) == (H, W) is OhemCrossEntropy2d at label resolution (standalone)
GEOMETRIES = [
    ((65, 129), (512, 1024), 8),       # the benchmark's DSN upsample
    ((65, 129), (512, 1024), 16),
    ((46, 61), (360, 480), 8),         # the last grid column reads 0 (zero column)
    ((5, 6), (36, 44), 8),             # grid size rounds half to even (4 x 6)
    ((3, 9), (11, 64), 8),             # a one-point grid axis (H < 1.5 factor)
    ((14, 17), (109, 131), 8),         # the last grid row rounds outside the image
    ((109, 131), (109, 131), 8),
    ((99, 131), (99, 131), 2),         # ratio exactly 2: every grid point on a pixel
    ((13, 17), (99, 131), 2),
    ((37, 45), (37, 45), 1),           # factor 1: the grid is the image
    ((13, 17), (37, 45), 1),
    ((97, 131), (97, 131), 4),
]


@pytest.fixture(scope="module")
def ops():
    from structure_knowledge_distillation_b200 import ops as o
    return o


def _rel(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _rel_scalar(a, b):
    a, b = float(torch.as_tensor(a).detach()), float(torch.as_tensor(b).detach())
    return abs(a - b) / max(abs(b), 1e-30) if b != 0 else abs(a)


def _edge(g, ref):
    """worst |g - ref| on the first / last row and column of the (N, C, h, w) gradient, over max |ref|"""
    d = (g.detach().double() - ref.detach().double()).abs()
    e = max(float(d[:, :, 0].max()), float(d[:, :, -1].max()), float(d[:, :, :, 0].max()), float(d[:, :, :, -1].max()))
    return e / max(float(ref.abs().max()), 1e-30)


def _layout(t, kind):
    """(N, C, H, W) float32 on the GPU as NCHW, channels-last, or a channel slice of an NHWC buffer pitched to a multiple of 4 with NaN
    in the pad channels (a multiple of 4 still gets 4 pad channels)"""
    t = t.float().cuda()
    if kind == "nchw":
        return t.contiguous()
    if kind == "nhwc":
        return t.contiguous(memory_format=torch.channels_last)
    n, c, h, w = t.shape
    pitch = (c + 3) // 4 * 4 if c % 4 else c + 4
    buf = torch.full((n, h, w, pitch), float("nan"), device="cuda")
    buf[..., :c] = t.permute(0, 2, 3, 1)
    return buf.permute(0, 3, 1, 2)[:, :c]


def _logits(g, shape, regime):
    """float64 logits that float32 holds exactly"""
    x = torch.randn(*shape, generator=g, device="cuda", dtype=torch.float64)
    scale, offset = dict(randn=(2.0, 0.0), peaked=(20.0, 0.0), offset=(2.0, 1e3))[regime]
    return (x * scale + offset).float().double()


def _labels(g, n, H, W, C, ignore_frac=0.05, ignore_index=255):
    lab = torch.randint(0, C, (n, H, W), generator=g, device="cuda")
    lab[torch.rand(n, H, W, generator=g, device="cuda") < ignore_frac] = ignore_index
    return lab


def _same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)


def _up(x, H, W):
    return F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)


def _prob(l0, H, W):
    return torch.softmax(_up(l0, H, W), 1)


def _max(t):
    return float(t.max()) if t.numel() else 0.0


def _merge(worst, rep):
    for k, v in rep.items():
        worst[k] = max(worst.get(k, 0.0), v)


# ------------------------------------------------------------------------------------------------ 1. grid sample
def _grid_case(ops, l64, labels, factor, ignore, kind, regime):
    H, W = labels.shape[1:]
    gh, gw = O.grid_shape(H, W, factor)
    runs = [ops.ohem_grid_sample(_layout(l64, kind), labels, factor, ignore, want_labels=True) for _ in range(2)]
    assert all(_same_bits(a, b) for a, b in zip(runs[0], runs[1])), "grid sample is not deterministic"
    pred, glab, nvalid = runs[0]
    ref, ref_lab = O.ohem_grid64(_prob(l64, H, W), labels, gh, gw, ignore)
    tag = (tuple(l64.shape), (H, W), factor, ignore, kind, regime)
    assert pred.shape == ref.shape == (l64.shape[0], gh, gw), tag
    assert torch.equal(glab, ref_lab), tag
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isinf(pred), ~fin) and (pred[~fin] > 0).all(), tag            # +inf exactly where ignored
    assert int(nvalid) == int(fin.sum()), tag
    assert torch.equal(pred[fin & (ref == 0)], torch.zeros_like(pred[fin & (ref == 0)])), tag  # points outside the image read 0
    v, r = pred[fin].double(), ref[fin]
    if regime == "randn":
        return dict(grid=_max((v - r).abs() / r.clamp_min(1e-30)))
    r32 = O.ohem_grid64(_prob(l64.float(), H, W).double(), labels, gh, gw, ignore)[0][fin].float().double()
    den = r.clamp_min(1e-6)
    e, e32 = _max((v - r).abs() / den), _max((r32 - r).abs() / den)
    assert e <= F32_FACTOR * e32 + PEAK_GRID_FLOOR, (tag, e, e32)
    return {"grid_" + regime: e, "f32_" + regime: e32}


@pytest.mark.parametrize("C", CLASSES)
def test_grid_sample_vs_float64(ops, C):
    """Every geometry with unit-scale, peaked and offset logits, each layout in turn; a custom ignore_index on the grid whose last row
    rounds outside the image (its label 0 is then ignored too when the ignore index is 0)."""
    g = torch.Generator(device="cuda").manual_seed(100 + C)
    worst = {}
    for gi, (hw, HW, factor) in enumerate(GEOMETRIES):
        for ri, regime in enumerate(("randn", "peaked", "offset")):
            l64 = _logits(g, (2, C) + hw, regime)
            labels = _labels(g, 2, *HW, C)
            rep = _grid_case(ops, l64, labels, factor, 255, LAYOUTS[(gi + ri) % 3], regime)
            if regime == "randn":
                assert rep["grid"] < GRID_TOL, ((hw, HW, factor, C), rep)
            _merge(worst, rep)
    for ignore in sorted({0, C // 2}):
        labels = _labels(g, 2, 109, 131, C, ignore_frac=0.0)
        labels[:, ::5] = ignore
        rep = _grid_case(ops, _logits(g, (2, C, 14, 17), "randn"), labels, 8, ignore, "pad4", "randn")
        assert rep["grid"] < GRID_TOL, ("ignore", ignore, rep)
        _merge(worst, rep)
    print("\nPARITY ohem_grid C=%d" % C, {k: "%.2e" % v for k, v in worst.items()})


def test_empty_grid_raises_before_launch(ops):
    """H < factor / 2: scipy's zoom gives an empty array, whose order statistic does not exist"""
    l0 = torch.randn(1, 19, 3, 9, device="cuda")
    labels = torch.randint(0, 19, (1, 3, 64), device="cuda")
    assert O.grid_shape(3, 64, 8)[0] == 0
    with pytest.raises(RuntimeError, match="skd_ohem_grid_sample"):
        ops.ohem_grid_sample(l0, labels, 8, 255)
    from structure_knowledge_distillation_b200 import functions as Fn
    with pytest.raises(RuntimeError, match="skd_ohem_grid_sample"):
        Fn.OhemDsnCrossEntropy.apply(l0.requires_grad_(True), None, labels, 255, 0.7, 1000, 8, 1.0, 0.0)


# ------------------------------------------------------------------------------------------------ 2. threshold
def _apply(l0, l1, labels, ignore, thresh, min_kept, factor, w0, w1):
    from structure_knowledge_distillation_b200 import functions as Fn
    return Fn.OhemDsnCrossEntropy.apply(l0, l1, labels, ignore, thresh, min_kept, factor, w0, w1)


@pytest.mark.parametrize("C", CLASSES)
def test_threshold_is_the_order_statistic_of_the_grid(ops, C):
    """The device threshold of OhemDsnCrossEntropy equals, bit for bit, ohem_threshold on the kernel's own grid values, on every
    branch: min_kept // f^2 >= valid (1.0), = valid - 1, = 1, = 0 (thresh), thresh equal to the order statistic, thresh above it,
    heavy ties among the grid values, and a batch with one image entirely ignored."""
    g = torch.Generator(device="cuda").manual_seed(300 + C)
    cases = [((65, 129), (512, 1024), 8, "randn"), ((13, 17), (37, 45), 1, "randn"), ((99, 131), (99, 131), 2, "ties"),
             ((14, 17), (109, 131), 8, "one_image_ignored")]
    seen = set()
    for hw, HW, f, kind in cases:
        if kind == "ties":                                          # integer logits: p[label] takes a handful of values
            l64 = torch.randint(-1, 2, (2, C) + hw, generator=g, device="cuda").double()
        else:
            l64 = _logits(g, (2, C) + hw, "randn")
        labels = _labels(g, 2, *HW, C)
        if kind == "one_image_ignored":
            labels[1] = 255
        l0, l1 = _layout(l64, "nhwc"), _layout(_logits(g, (2, C) + hw, "randn"), "pad4")
        pred, _, nvalid = ops.ohem_grid_sample(l0, labels, f, 255)
        nv = int(nvalid)
        vals = pred[torch.isfinite(pred)].sort().values
        p = pred.cpu().numpy()
        if kind == "ties":
            assert vals.unique().numel() <= nv // 3, vals.unique().numel()
        mid = vals[nv // 2].item()
        for k, thresh in ((nv + 3, 0.0), (nv, 0.0), (nv - 1, 0.0), (1, 0.0), (0, 0.7), (0, 0.0), (nv // 2 + 1, mid),
                          (nv // 3 + 1, 0.7), (nv // 2 + 1, 0.0)):
            _, thr, _ = _apply(l0, l1, labels, 255, thresh, k * f * f, f, 1.0, 0.4)
            want = torch.tensor(O.ohem_threshold(p, k, thresh), dtype=torch.float32)
            assert _same_bits(thr.cpu(), want), (C, hw, HW, f, kind, k, thresh, float(thr), float(want))
            seen.add("one" if float(want) == 1.0 else "thresh" if float(want) == float(torch.tensor(thresh).float()) else "kth")
    assert seen == {"one", "thresh", "kth"} or C == 1, seen
    print("\nPARITY ohem_threshold C=%d" % C, sorted(seen), "bit-identical")


# ------------------------------------------------------------------------------------------------ 3. masked loss and gradients
def _ohem_ops(ops, ls, labels, ignore, thresh, min_kept, factor, w0, w1):
    """the pipeline of OhemDsnCrossEntropy through ops (for both counts), twice and bit-identical, and equal bit for bit to the
    autograd function -> (thr, loss, counts, grads, pred)"""
    H = labels.shape[1]
    l0, l1 = ls[0], (ls[1] if len(ls) == 2 else None)
    res = []
    for _ in range(2):
        pred, _, nvalid = ops.ohem_grid_sample(l0, labels, factor, ignore)
        thr = ops.ohem_threshold(pred, nvalid, min_kept // (factor * factor), thresh)
        loss, counts, rows = ops.ohem_dsn_ce_fwd_train(l0, l1, labels, ignore, w0, w1, thr)
        d0, d1 = ops.ohem_dsn_ce_bwd_cols(l0, l1, rows, H, w0, w1, torch.ones((), device="cuda"), counts)
        res.append((thr, loss, counts, (d0,) if l1 is None else (d0, d1), pred))
    a, b = res
    assert all(_same_bits(x, y) for x, y in zip(a[:3], b[:3])) and all(_same_bits(x, y) for x, y in zip(a[3], b[3])), \
        "OHEM is not deterministic"
    x = [t.detach().requires_grad_(True) for t in ls]
    loss, thr, kept = _apply(x[0], x[1] if len(x) == 2 else None, labels, ignore, thresh, min_kept, factor, w0, w1)
    grads = torch.autograd.grad(loss, x)
    assert _same_bits(thr, a[0]) and _same_bits(loss.detach(), a[1]) and float(kept) == float(a[2][0])
    assert all(_same_bits(p, q) for p, q in zip(grads, a[3])), "OhemDsnCrossEntropy and the ops differ"
    return a


def _grid_pixels(H, W, gh, gw, device):
    """-> (nearest-neighbour sources of the grid labels, pixels that ARE a grid point, and that point's (gy, gx) per pixel), (H, W)"""
    y0, _, ty, _, ny, oy = O.zoom_axis64(H, gh, device)
    x0, _, tx, _, nx, ox = O.zoom_axis64(W, gw, device)
    nn = torch.zeros(H, W, dtype=torch.bool, device=device)
    nn[ny[~oy][:, None], nx[~ox]] = True
    on = torch.zeros(H, W, dtype=torch.bool, device=device)
    at = torch.zeros(2, H, W, dtype=torch.long, device=device)
    iy, ix = (ty == 0) & ~oy, (tx == 0) & ~ox
    on[y0[iy][:, None], x0[ix]] = True
    at[0][y0[iy][:, None], x0[ix]] = torch.arange(gh, device=device)[iy][:, None]
    at[1][y0[iy][:, None], x0[ix]] = torch.arange(gw, device=device)[ix]
    return nn, on, at


def _masked_check(ops, l64, labels, factor, ignore=255, thresh=0.0, keep_frac=0.5, weights=(1.0, 0.4), layouts=("nchw", "nchw"),
                  regime="randn", tag=()):
    """OHEM on head 0 against float64 at the kernel's threshold; -> report of errors"""
    heads = len(l64)
    n, C = l64[0].shape[:2]
    H, W = labels.shape[1:]
    gh, gw = O.grid_shape(H, W, factor)
    ls = [_layout(t, k) for t, k in zip(l64, layouts)]
    w0, w1 = weights
    nv = int(ops.ohem_grid_sample(ls[0], labels, factor, ignore)[2])
    min_kept = max(1, int(nv * keep_frac)) * factor * factor
    thr = _ohem_ops(ops, ls, labels, ignore, thresh, min_kept, factor, w0, w1)[0]
    t = float(thr)
    # pixels too close to the threshold to decide in float64: ignored, unless a grid label comes from them
    valid = labels != ignore
    prob = _prob(l64[0], H, W)
    p64 = prob.gather(1, torch.where(valid, labels, 0).clamp(0, C - 1)[:, None])[:, 0]
    nn, on, at = _grid_pixels(H, W, gh, gw, labels.device)
    close = valid & ((p64 - t).abs() <= UNDECIDED[regime] * t) & (t < 1.0)          # (p <= 1 holds in any precision)
    labels = labels.clone()
    labels[close & ~nn] = ignore
    thr2, loss, counts, grads, pred = _ohem_ops(ops, ls, labels, ignore, thresh, min_kept, factor, w0, w1)
    assert _same_bits(thr2, thr), (tag, "threshold moved", t, float(thr2))
    left = close & nn
    keep = valid & (labels != ignore) & (p64 <= t)
    if left.any():                      # a pixel that is a grid point: its probability is that point's value, kept iff <= thr
        nidx = torch.arange(n, device=labels.device)[:, None, None].expand(n, H, W)
        keep = torch.where(left & on, pred[nidx, at[0], at[1]] <= thr2, keep)
    # an undecidable pixel that only feeds a grid label (rare: a few per million pixels) keeps the kernel's own decision, read from
    # the masked forward at the same threshold on a label map holding that pixel alone
    alone = (left & ~on).nonzero().tolist()
    assert len(alone) <= 4, (tag, "too many undecidable grid-label pixels", len(alone))
    for i, y, x in alone:
        one = torch.full_like(labels, ignore)
        one[i, y, x] = labels[i, y, x]
        keep[i, y, x] = float(ops.ohem_dsn_ce_fwd_train(ls[0], None, one, ignore, 1.0, 0.0, thr2)[1][0]) > 0
    masked = torch.where(keep, labels, ignore)
    valid1 = int((labels != ignore).sum())
    assert int(counts[0]) == int(keep.sum()), (tag, "kept", int(counts[0]), int(keep.sum()))
    assert int(counts[1]) == (valid1 if heads == 2 else 0), (tag, "head-1 valid", int(counts[1]), valid1)

    def ref_of(xs):
        r = w0 * F.cross_entropy(_up(xs[0], H, W), masked, ignore_index=ignore)
        if heads == 2:
            r = r + w1 * F.cross_entropy(_up(xs[1], H, W), labels, ignore_index=ignore)
        return r, torch.autograd.grad(r, xs)

    ref, gref = ref_of([t64.clone().requires_grad_(True) for t64 in l64])
    rep = dict(loss=_rel_scalar(loss, ref), grad=max(_rel(a, b) for a, b in zip(grads, gref)),
               edge=max(_edge(a, b) for a, b in zip(grads, gref)))
    if regime == "randn":
        assert rep["loss"] < LOSS_TOL and rep["grad"] < GRAD_TOL and rep["edge"] < EDGE_TOL, (tag, rep)
    else:
        r32, g32 = ref_of([t64.float().requires_grad_(True) for t64 in l64])
        e32 = dict(loss=_rel_scalar(r32, ref), grad=max(_rel(a, b) for a, b in zip(g32, gref)),
                   edge=max(_edge(a, b) for a, b in zip(g32, gref)))
        assert rep["loss"] <= F32_FACTOR * e32["loss"] + PEAK_LOSS_FLOOR, (tag, rep, e32)
        assert rep["grad"] <= F32_FACTOR * e32["grad"] + PEAK_GRAD_FLOOR, (tag, rep, e32)
        assert rep["edge"] <= F32_FACTOR * e32["edge"] + PEAK_GRAD_FLOOR, (tag, rep, e32)
        rep = {k + "_" + regime: v for k, v in rep.items()}
    rep["kept_frac"] = float(counts[0]) / max(valid1, 1)
    rep["undecided"] = float(close.sum())
    return rep


@pytest.mark.parametrize("C", CLASSES)
def test_masked_loss_class_counts(ops, C):
    """Both row-kernel instantiations (CT = 19, 32), one and two heads, w1 = 0, every layout, unit-scale, peaked and offset logits,
    on a (13, 17) -> (97, 131) upsample at factor 8, the threshold at the median grid value."""
    g = torch.Generator(device="cuda").manual_seed(500 + C)
    worst = {}
    cases = [(2, "randn", (1.0, 0.4)), (1, "randn", (1.0, 0.0)), (2, "randn", (1.0, 0.0)), (2, "peaked", (1.0, 0.4)),
             (1, "offset", (1.0, 0.0))]
    lays = [("nchw", "nhwc"), ("pad4", "nchw"), ("nhwc", "pad4")]
    for k, (heads, regime, weights) in enumerate(cases):
        l64 = [_logits(g, (2, C, 13, 17), regime) for _ in range(heads)]
        labels = _labels(g, 2, 97, 131, C)
        for lay in ([lays[k % 3]] if regime != "randn" else lays):
            _merge(worst, _masked_check(ops, l64, labels, 8, weights=weights, layouts=lay, regime=regime,
                                        tag=(C, heads, regime, weights, lay)))
    print("\nPARITY ohem_masked C=%d" % C, {k: "%.2e" % v for k, v in worst.items()})


@pytest.mark.parametrize("C", [19, 32])
@pytest.mark.parametrize("hw,HW,factor", GEOMETRIES + [((9, 129), (16, 1500), 4)])
def test_masked_loss_geometries(ops, hw, HW, factor, C):
    """Every grid geometry, and a label width above 1 024 (the row phase in two column chunks), DSN with two heads and standalone."""
    g = torch.Generator(device="cuda").manual_seed(hw[0] * 1000 + HW[1] * 10 + factor + C)
    heads, lay = (1, ("pad4",)) if hw == HW else (2, ("nhwc", "pad4"))
    l64 = [_logits(g, (2, C) + hw, "randn") for _ in range(heads)]
    labels = _labels(g, 2, *HW, C)
    rep = _masked_check(ops, l64, labels, factor, weights=(1.0, 0.4) if heads == 2 else (1.0, 0.0), layouts=lay,
                        tag=(hw, HW, factor, C))
    print("\nPARITY ohem_masked %s->%s f=%d C=%d" % (hw, HW, factor, C), {k: "%.2e" % v for k, v in rep.items()})


def test_masked_loss_custom_ignore_index_and_thresh(ops):
    """A class id as ignore_index, and the threshold set by thresh (above the order statistic)"""
    g = torch.Generator(device="cuda").manual_seed(77)
    l64 = [_logits(g, (2, 19, 14, 17), "randn") for _ in range(2)]
    labels = _labels(g, 2, 109, 131, 19, ignore_frac=0.0)
    rep = _masked_check(ops, l64, labels, 8, ignore=3, layouts=("pad4", "nhwc"), tag="ignore 3")
    rep2 = _masked_check(ops, l64, labels, 8, thresh=0.1, keep_frac=0.05, layouts=("nhwc", "nchw"), tag="thresh 0.1")
    print("\nPARITY ohem_masked ignore=3", {k: "%.2e" % v for k, v in rep.items()}, "thresh=0.1",
          {k: "%.2e" % v for k, v in rep2.items()})


# ------------------------------------------------------------------------------------------------ 4. the pixel at the threshold
@pytest.mark.parametrize("mode", ["standalone_f1", "dsn_f1", "standalone_f2", "dsn_f2"])
def test_pixel_at_the_threshold_is_kept(ops, mode):
    """Where every valid pixel is a grid point (factor 1; factor 2 at 99 x 131 with the labels off the even rows and columns
    ignored), the reference thresholds the very probabilities it ranked: kept = #{valid grid values <= thr}, which is min_kept when
    the values are distinct.  The grid and the mask must compute a pixel's probability the same way for this to hold."""
    dsn, f = mode.startswith("dsn"), int(mode[-1])
    HW = (37, 45) if f == 1 else (99, 131)
    hw = (13, 17) if dsn else HW
    wrong, total = [], 0
    for seed in range(3):
        for C in (19, 32):
            g = torch.Generator(device="cuda").manual_seed(seed * 100 + C + f)
            l0 = _layout(_logits(g, (2, C) + hw, "randn"), "nhwc")
            l1 = _layout(_logits(g, (2, C) + hw, "randn"), "nchw") if dsn else None
            labels = _labels(g, 2, *HW, C)
            if f == 2:
                labels[:, 1::2] = 255
                labels[:, :, 1::2] = 255
            pred, _, nvalid = ops.ohem_grid_sample(l0, labels, f, 255)
            nv = int(nvalid)
            vals = pred[torch.isfinite(pred)]
            assert int((labels != 255).sum()) == nv
            for k in (1, 2, nv // 7, nv // 3, nv // 2, nv - 1):
                _, thr, kept = _apply(l0, l1, labels, 255, 0.0, k * f * f, f, 1.0, 0.4 if dsn else 0.0)
                want = int((vals <= thr).sum())
                if vals.unique().numel() == nv:
                    assert want == k
                total += 1
                if int(kept) != want:
                    wrong.append((seed, C, k, int(kept), want))
    print("\nPARITY ohem_tie %s: %d of %d cases wrong (seed, C, min_kept, kept, expected): %s" % (mode, len(wrong), total, wrong))
    assert not wrong


# ------------------------------------------------------------------------------------------------ 5. degenerate equalities
@pytest.mark.parametrize("C", CLASSES[1:])
def test_threshold_one_equals_dsn_cross_entropy(ops, C):
    """min_kept above the valid count: threshold 1.0 keeps every valid pixel, and CriterionOhemDSN is CriterionDSN -- the same row and
    column kernels with equal denominators give bit-identical gradients, and the loss (one division per head instead of one for
    both) agrees within 2 ulp."""
    from structure_knowledge_distillation_b200 import functions as Fn
    g = torch.Generator(device="cuda").manual_seed(700 + C)
    for heads, lay in ((2, ("nhwc", "pad4")), (1, ("pad4",))):
        l64 = [_logits(g, (2, C, 13, 17), "randn") for _ in range(heads)]
        labels = _labels(g, 2, 97, 131, C)
        w1 = 0.4 if heads == 2 else 0.0
        xs = [_layout(t, k).requires_grad_(True) for t, k in zip(l64, lay)]
        l1 = xs[1] if heads == 2 else None
        loss, thr, kept = _apply(xs[0], l1, labels, 255, 0.7, 10 ** 9, 8, 1.0, w1)
        go = torch.autograd.grad(loss, xs)
        plain = Fn.DsnCrossEntropy.apply(xs[0], l1, labels, 255, 1.0, w1)
        gp = torch.autograd.grad(plain, xs)
        assert float(thr) == 1.0 and int(kept) == int((labels != 255).sum())
        assert all(_same_bits(a, b) for a, b in zip(go, gp)), (C, heads)
        ulp = torch.finfo(torch.float32).eps * abs(float(plain))
        assert abs(float(loss) - float(plain)) <= 2 * ulp, (C, heads, float(loss), float(plain))


def test_one_class_keeps_everything_at_zero_loss(ops):
    """C = 1: p[label] = 1 everywhere, so the threshold is 1.0 whatever min_kept, every valid pixel is kept, and loss and gradient are 0"""
    g = torch.Generator(device="cuda").manual_seed(9)
    for hw, HW, f in (((13, 17), (97, 131), 8), ((37, 45), (37, 45), 1)):
        x0 = _layout(_logits(g, (2, 1) + hw, "randn"), "pad4").requires_grad_(True)
        x1 = _layout(_logits(g, (2, 1) + hw, "randn"), "nchw").requires_grad_(True)
        labels = _labels(g, 2, *HW, 1)
        for mk in (f * f, 100 * f * f):
            loss, thr, kept = _apply(x0, x1, labels, 255, 0.0, mk, f, 1.0, 0.4)
            g0, g1 = torch.autograd.grad(loss, [x0, x1])
            assert float(thr) == 1.0 and int(kept) == int((labels != 255).sum()) and float(loss) == 0.0, (hw, mk)
            assert float(g0.abs().max()) == 0.0 and float(g1.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ 6. width limit
def _rows_smem_bytes(C, w, W):
    """dsn_rows_launch's shared memory: the softmax chunk [C][chunk | 1], two weight rows, the run starts and one blended row"""
    chunk = min(W, 1024)
    return (C * (chunk | 1) + 2 * chunk + w + 2 + w * C) * 4


@pytest.mark.parametrize("C,expected", [(19, 1483), (32, 763)])
def test_standalone_width_limit(ops, C, expected):
    """OhemCrossEntropy2d at label resolution holds one row of logits in shared memory: the widest input that fits runs and matches
    float64, one column more raises instead of launching."""
    limit = max(W for W in range(1, 4096) if _rows_smem_bytes(C, W, W) <= 200 * 1024)
    assert limit == expected
    g = torch.Generator(device="cuda").manual_seed(C)
    l64 = [_logits(g, (1, C, 8, limit), "randn")]
    labels = _labels(g, 1, 8, limit, C)
    rep = _masked_check(ops, l64, labels, 4, layouts=("pad4",), tag=("width", C, limit))
    print("\nPARITY ohem_width C=%d W=%d" % (C, limit), {k: "%.2e" % v for k, v in rep.items()})
    x = torch.randn(1, C, 8, limit + 1, device="cuda", requires_grad=True)
    with pytest.raises(RuntimeError, match="source width too large"):
        _apply(x, None, torch.randint(0, C, (1, 8, limit + 1), device="cuda"), 255, 0.7, 1000, 4, 1.0, 0.0)
