"""The loss kernels of csrc/losses.cu against float64 torch over the shapes, class counts, label geometries and layouts where they can
go wrong: pixel-wise (Pi), the DSN cross entropy through its three entry paths (eval forward, fused training forward + column phase,
unfused backward), and the SIMT pair-wise path (Pa).

The float64 references are oracle/port.py's restatements (pinned against the unmodified reference in test_oracle_golden.py), run on the
GPU.  The same references in float32 torch measure the reference's own precision where the logits are sharply peaked.  Every case runs
twice and must give bit-identical results (the wgmma Pa path excepted: its loss reduction adds doubles atomically, DESIGN.md §6)."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import port

pytestmark = pytest.mark.gpu

CLASSES = [1, 2, 3, 4, 7, 19, 20, 21, 31, 32]
# bounds about 5x the worst error measured on an H100 (DESIGN.md §4)
LOSS_TOL = 2e-6            # relative, losses against float64
GRAD_TOL = 2e-5            # rel-L2, gradients against float64
EDGE_TOL = 2e-5            # worst element on the first / last logit row and column, relative to the largest gradient element
# peaked logits (randn * 20), and the pair-wise gradient away from zero nodes: the kernel's error may be 4x float32 torch's plus a
# floor.  A one-pixel softmax difference of two nearly one-hot rows cancels to ~1e-17, where float32 torch is as far off (rel-L2 ~0.7)
# as the kernel.  On such tiny single-pixel losses the pixel-wise kernel's relative error reaches a few 1e-6, up to 13.6x float32
# torch's; with expf / logf in place of __expf / __logf it is still up to 9x, so the floor, not the intrinsics, is what they need
F32_FACTOR = 4.0
PEAK_LOSS_FLOOR = 1e-5
PEAK_GRAD_FLOOR = 1e-4


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
    in the pad channels (the pad4 carriers of the 19 / 21-class logits; a multiple of 4 still gets 4 pad channels)"""
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
    x = torch.randn(*shape, generator=g, device="cuda", dtype=torch.float64)
    if regime == "randn":
        return x * 2
    if regime == "peaked":
        return x * 20
    if regime == "offset":
        return x * 2 + 1e3
    raise ValueError(regime)


def _same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)


# ------------------------------------------------------------------------------------------------ pixel-wise
PI_SIZES = [(1, 1, 1), (2, 13, 17), (3, 1, 33), (8, 65, 129)]
PI_LAYOUTS = [("nchw", "nchw"), ("nhwc", "pad4"), ("pad4", "nchw"), ("nhwc", "nhwc")]


def _pi_case(ops, S64, T64, ls, lt):
    from structure_knowledge_distillation_b200.utils.criterion import CriterionPixelWise
    out = []
    for _ in range(2):
        S = _layout(S64, ls).requires_grad_(True)
        T = _layout(T64, lt)
        loss = CriterionPixelWise()([S], [T])
        (g,) = torch.autograd.grad(loss, S)
        out.append((loss.detach(), g))
        # the ops directly, with a non-unit upstream gradient
        assert _same_bits(ops.pixelwise_fwd(S.detach(), T), loss.detach())
        g3 = ops.pixelwise_bwd(S.detach(), T, torch.full((), 3.0, device="cuda"))
        assert torch.allclose(g3, 3 * g, rtol=1e-6, atol=1e-6 * float(g3.abs().max()))   # (peaked rows reach subnormals)
    assert _same_bits(out[0][0], out[1][0]) and _same_bits(out[0][1], out[1][1]), "pixel-wise is not deterministic"
    return out[0]


@pytest.mark.parametrize("C", CLASSES)
def test_pixelwise_vs_float64(ops, C):
    g = torch.Generator(device="cuda").manual_seed(1000 + C)
    worst = dict(loss=0.0, grad=0.0, edge=0.0, peaked_loss_ratio=0.0, peaked_grad_ratio=0.0)
    for n, h, w in PI_SIZES:
        for r, regime in enumerate(("randn", "peaked", "offset", "same")):
            # every layout pair on the small sizes, one per regime (in turn) on the largest
            for ls, lt in ([PI_LAYOUTS[r]] if n * h * w > 1000 else PI_LAYOUTS):
                S64 = _logits(g, (n, C, h, w), "randn" if regime == "same" else regime).float().double()
                T64 = S64.clone() if regime == "same" else _logits(g, (n, C, h, w), regime).float().double()
                loss, grad = _pi_case(ops, S64, T64, ls, lt)
                Sd = S64.clone().requires_grad_(True)
                ref = port.pixelwise_loss(Sd, T64)
                (gref,) = torch.autograd.grad(ref, Sd)
                tag = (C, n, h, w, regime, ls, lt)
                assert torch.isfinite(loss) and torch.isfinite(grad).all(), tag
                if C == 1:                                             # one class: log 1 - 0, exactly
                    assert float(loss) == 0.0 and float(grad.abs().max()) == 0.0, tag
                    continue
                e_loss = _rel_scalar(loss, ref)
                # the gradient is (softmax(S) - softmax(T)) / (h w): every row sums to 0
                assert float(grad.double().sum(1).abs().max()) < 1e-6 * C / (h * w), tag
                if regime == "same":
                    # S == T: the loss is the teacher's entropy and the gradient vanishes up to float32 rounding of the probabilities
                    assert e_loss < LOSS_TOL, (tag, e_loss)
                    assert float(grad.abs().max()) < 1e-6 / (h * w), tag
                    continue
                e_grad, e_edge = _rel(grad, gref), _edge(grad, gref)
                if regime != "peaked":
                    worst["loss"] = max(worst["loss"], e_loss); worst["grad"] = max(worst["grad"], e_grad)
                    worst["edge"] = max(worst["edge"], e_edge)
                if regime == "peaked":
                    # yardstick: the same reference in float32 torch
                    S32 = S64.float().requires_grad_(True)
                    r32 = port.pixelwise_loss(S32, T64.float())
                    (g32,) = torch.autograd.grad(r32, S32)
                    e32_loss, e32_grad = _rel_scalar(r32, ref), _rel(g32, gref)
                    worst["peaked_loss_ratio"] = max(worst["peaked_loss_ratio"], e_loss / max(e32_loss, 1e-12))
                    worst["peaked_grad_ratio"] = max(worst["peaked_grad_ratio"], e_grad / max(e32_grad, 1e-12))
                    assert e_loss <= F32_FACTOR * e32_loss + PEAK_LOSS_FLOOR, (tag, e_loss, e32_loss)
                    assert e_grad <= F32_FACTOR * e32_grad + PEAK_GRAD_FLOOR, (tag, e_grad, e32_grad)
                    assert e_edge <= F32_FACTOR * _edge(g32, gref) + PEAK_GRAD_FLOOR, tag
                else:
                    assert e_loss < LOSS_TOL and e_grad < GRAD_TOL and e_edge < EDGE_TOL, (tag, e_loss, e_grad, e_edge)
    print("\nPARITY pixelwise C=%d" % C, {k: "%.2e" % v for k, v in worst.items()})


# ------------------------------------------------------------------------------------------------ DSN cross entropy
def _ce_ref(preds, weights, labels, ignore_index):
    """port.dsn_ce_loss (CriterionDSN: weights 1.0 / 0.4) and its single-head form (CriterionCrossEntropy)"""
    if len(preds) == 2 and weights == (1.0, 0.4):
        return port.dsn_ce_loss(preds, labels, ignore_index)
    H, W = labels.shape[1:]
    up = F.interpolate(preds[0], size=(H, W), mode="bilinear", align_corners=True)
    return F.cross_entropy(up, labels, ignore_index=ignore_index)


def _dsn_paths(ops, l64, labels, ignore_index, weights, layouts):
    """-> {path: (loss, grads)} for the eval forward (loss only), the fused training forward + column phase, and the unfused backward;
    each run twice, bit-identical"""
    from structure_knowledge_distillation_b200 import functions as Fn
    w0, w1 = weights
    res = []
    for _ in range(2):
        ls = [_layout(t, kind) for t, kind in zip(l64, layouts)]
        l0, l1 = ls[0], (ls[1] if len(ls) == 2 else None)
        ev = ops.dsn_ce_fwd(l0, l1, labels, ignore_index, w0, w1)
        x = [t.detach().requires_grad_(True) for t in ls]
        loss = Fn.DsnCrossEntropy.apply(x[0], x[1] if len(x) == 2 else None, labels, ignore_index, w0, w1)
        fused = torch.autograd.grad(loss, x)
        d0, d1 = ops.dsn_ce_bwd(l0, l1, labels, ignore_index, w0, w1, torch.ones((), device="cuda"), ev[1])
        unfused = (d0,) if l1 is None else (d0, d1)
        res.append(dict(eval=ev[0].clone(), count=ev[1].clone(), train=loss.detach(), fused=fused, unfused=unfused))
    a, b = res
    for k in ("eval", "count", "train"):
        assert _same_bits(a[k], b[k]), "DSN %s is not deterministic" % k
    for k in ("fused", "unfused"):
        assert all(_same_bits(p, q) for p, q in zip(a[k], b[k])), "DSN %s gradient is not deterministic" % k
    # the training forward's row phase and the unfused backward's are the same kernel code: the gradients agree bit for bit
    assert all(_same_bits(p, q) for p, q in zip(a["fused"], a["unfused"])), "fused and unfused DSN gradients differ"
    return a


def _dsn_check(ops, l64, labels, ignore_index=255, weights=(1.0, 0.4), layouts=("nchw", "nchw"), peaked=False, tag=()):
    heads = len(l64)
    a = _dsn_paths(ops, l64, labels, ignore_index, weights, layouts[:heads])
    xd = [t.clone().requires_grad_(True) for t in l64]
    ref = _ce_ref(xd, weights, labels, ignore_index)
    gref = torch.autograd.grad(ref, xd)
    nvalid = int((labels != ignore_index).sum())
    assert float(a["count"]) == nvalid, (tag, float(a["count"]), nvalid)
    rep = dict(eval=_rel_scalar(a["eval"], ref), train=_rel_scalar(a["train"], ref), eval_vs_train=_rel_scalar(a["eval"], a["train"]),
               grad=max(_rel(g, r) for g, r in zip(a["fused"], gref)), edge=max(_edge(g, r) for g, r in zip(a["fused"], gref)))
    # the eval forward interpolates the four logits of a pixel directly, the training forward blends each source row pair first and
    # sums in another order: the two losses differ only by float32 rounding
    assert rep["eval_vs_train"] < 1e-6, (tag, rep)
    if peaked:
        x32 = [t.float().requires_grad_(True) for t in l64]
        r32 = _ce_ref(x32, weights, labels, ignore_index)
        g32 = torch.autograd.grad(r32, x32)
        e32 = dict(loss=_rel_scalar(r32, ref), grad=max(_rel(g, r) for g, r in zip(g32, gref)),
                   edge=max(_edge(g, r) for g, r in zip(g32, gref)))
        bound = F32_FACTOR * e32["loss"] + PEAK_LOSS_FLOOR
        assert rep["eval"] <= bound and rep["train"] <= bound, (tag, rep, e32)
        assert rep["grad"] <= F32_FACTOR * e32["grad"] + PEAK_GRAD_FLOOR, (tag, rep, e32)
        assert rep["edge"] <= F32_FACTOR * e32["edge"] + PEAK_GRAD_FLOOR, (tag, rep, e32)
        rep["f32_loss"], rep["f32_grad"] = e32["loss"], e32["grad"]
    else:
        assert rep["eval"] < LOSS_TOL and rep["train"] < LOSS_TOL, (tag, rep)
        assert rep["grad"] < GRAD_TOL and rep["edge"] < EDGE_TOL, (tag, rep)
    return rep


def _labels(g, n, H, W, C, ignore_frac=0.05, ignore_index=255):
    lab = torch.randint(0, C, (n, H, W), generator=g, device="cuda")
    lab[torch.rand(n, H, W, generator=g, device="cuda") < ignore_frac] = ignore_index
    return lab


def _merge(worst, rep):
    for k, v in rep.items():
        worst[k] = max(worst.get(k, 0.0), v)


@pytest.mark.parametrize("C", CLASSES)
def test_dsn_ce_class_counts(ops, C):
    """Every class count of the CT = 19 and CT = 32 instantiations (19 / 20 is the switch), one and two heads, every layout, unit-scale
    and peaked logits, on a (13, 17) -> (97, 131) upsample."""
    g = torch.Generator(device="cuda").manual_seed(2000 + C)
    worst = {}
    lays = [("nchw", "nhwc"), ("pad4", "nchw"), ("nhwc", "pad4")]
    for k, (heads, regime) in enumerate([(2, "randn"), (1, "randn"), (2, "peaked"), (1, "peaked")]):
        l64 = [_logits(g, (2, C, 13, 17), regime).float().double() for _ in range(heads)]
        labels = _labels(g, 2, 97, 131, C)
        weights = (1.0, 0.4) if heads == 2 else (1.0, 0.0)
        for lay in lays:
            _merge(worst, _dsn_check(ops, l64, labels, weights=weights, layouts=lay, peaked=regime == "peaked",
                                     tag=(C, heads, regime, lay)))
    print("\nPARITY dsn_ce C=%d" % C, {k: "%.2e" % v for k, v in worst.items()})


DSN_GEOMETRIES = [((65, 129), (512, 1024)), ((41, 41), (321, 321)), ((46, 61), (360, 480)), ((13, 17), (97, 131)),
                  ((360, 480), (360, 480)), ((1, 17), (97, 131)), ((13, 1), (97, 131)), ((13, 17), (1, 131)),
                  ((9, 129), (16, 1500))]


@pytest.mark.parametrize("C", [19, 20])
@pytest.mark.parametrize("hw,HW", DSN_GEOMETRIES)
def test_dsn_ce_geometries(ops, hw, HW, C):
    """The benchmark and VOC upsamples, same-size logits (the full ESPNet), one-row / one-column logits and labels (sy = 0 / sx = 0),
    and a label width above 1 024 (the row phase in two column chunks)."""
    g = torch.Generator(device="cuda").manual_seed(hw[0] * 1000 + HW[1] + C)
    n = 2
    worst = {}
    if hw == HW:                                                   # same size: the full ESPNet's single head, 360 x 480 in a 1024 row
        cases = [(1, ("nhwc",))]
    else:
        cases = [(2, ("nhwc", "pad4")), (1, ("pad4",))]
    for heads, lay in cases:
        l64 = [_logits(g, (n, C) + hw, "randn").float().double() for _ in range(heads)]
        labels = _labels(g, n, *HW, C)
        _merge(worst, _dsn_check(ops, l64, labels, weights=(1.0, 0.4) if heads == 2 else (1.0, 0.0), layouts=lay + lay,
                                 tag=(hw, HW, C, heads)))
    print("\nPARITY dsn_ce %s->%s C=%d" % (hw, HW, C), {k: "%.2e" % v for k, v in worst.items()})


@pytest.mark.parametrize("pattern", ["random", "rows", "one_image", "custom_index"])
def test_dsn_ce_ignore_patterns(ops, pattern):
    g = torch.Generator(device="cuda").manual_seed(31)
    C, n, hw, HW = 19, 2, (41, 41), (321, 321)
    ignore = 255
    labels = _labels(g, n, *HW, C, ignore_frac=0.05 if pattern == "random" else 0.0)
    if pattern == "rows":
        labels[:, ::3] = ignore
        labels[:, -1] = ignore
        labels[:, 0] = ignore
    elif pattern == "one_image":
        labels[1] = ignore
    elif pattern == "custom_index":                                # a class id as ignore_index: its pixels drop out, 255 is a label
        ignore = 3
    worst = {}
    for heads in (2, 1):
        l64 = [_logits(g, (n, C) + hw, "randn").float().double() for _ in range(heads)]
        _merge(worst, _dsn_check(ops, l64, labels, ignore_index=ignore, weights=(1.0, 0.4) if heads == 2 else (1.0, 0.0),
                                 layouts=("nhwc", "nchw"), tag=(pattern, heads)))
    print("\nPARITY dsn_ce ignore=%s" % pattern, {k: "%.2e" % v for k, v in worst.items()})


def test_dsn_ce_all_ignored_nan_loss_zero_gradient(ops):
    """Every label ignore_index: torch's cross entropy gives a NaN loss and an all-zero gradient.  CriterionDSN and
    CriterionCrossEntropy, fused (training forward + column phase) and unfused (eval forward + skd_dsn_ce_bwd), do the same: a 0/0
    denominator must not turn into NaN gradients that reach every parameter."""
    from structure_knowledge_distillation_b200.utils.criterion import CriterionCrossEntropy, CriterionDSN
    labels = torch.full((2, 97, 131), 255, device="cuda", dtype=torch.int64)
    for crit, heads in ((CriterionDSN(), 2), (CriterionCrossEntropy(), 1)):
        x = [torch.randn(2, 19, 13, 17, device="cuda", requires_grad=True) for _ in range(heads)]
        ref = _ce_ref([t.detach().double().requires_grad_(True) for t in x], (1.0, 0.4) if heads == 2 else (1.0, 0.0), labels, 255)
        assert torch.isnan(ref)
        loss = crit(x + [None] * (2 - heads), labels)
        grads = torch.autograd.grad(loss, x)
        assert torch.isnan(loss), type(crit).__name__
        for gr in grads:
            assert torch.equal(gr, torch.zeros_like(gr)), type(crit).__name__
        l1 = x[1].detach() if heads == 2 else None
        ev = ops.dsn_ce_fwd(x[0].detach(), l1, labels, 255, 1.0, 0.4 if heads == 2 else 0.0)
        assert torch.isnan(ev[0]) and float(ev[1]) == 0
        d0, d1 = ops.dsn_ce_bwd(x[0].detach(), l1, labels, 255, 1.0, 0.4 if heads == 2 else 0.0, torch.ones((), device="cuda"), ev[1])
        for gr in (d0, d1) if heads == 2 else (d0,):
            assert torch.equal(gr, torch.zeros_like(gr)), type(crit).__name__
    # one image of the batch all ignored: finite loss, and that image's gradient is exactly 0
    lab2 = _labels(torch.Generator(device="cuda").manual_seed(5), 2, 97, 131, 19)
    lab2[0] = 255
    x = torch.randn(2, 19, 13, 17, device="cuda", requires_grad=True)
    loss = CriterionCrossEntropy()([x, None], lab2)
    (gx,) = torch.autograd.grad(loss, x)
    assert torch.isfinite(loss) and torch.equal(gx[0], torch.zeros_like(gx[0])) and float(gx[1].abs().max()) > 0


@pytest.mark.parametrize("student,graph", [("resnet18", False), ("espnet_c", False), ("resnet18", True), ("espnet_c", True)])
def test_netmodel_step_on_all_ignored_batch_keeps_parameters_finite(student, graph):
    """A batch whose crops lie entirely in void pixels: the task loss is NaN, the step still updates the student from the distillation
    terms, and no parameter becomes NaN.  With CUDA graphs the step is captured on a batch with valid labels and the void batch is
    replayed through the same graph, so the zero count is handled on the device."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    m = NetModel(make_args(batch_size=2, pi=True, pa=True, ho=False, student=student))
    images = torch.randn(2, 3, 64, 96)
    labels = torch.full((2, 64, 96), 255, dtype=torch.int64)
    if graph:
        m.enable_cuda_graphs(warmup=1)
        valid = torch.randint(0, 19, (2, 64, 96))
        for _ in range(2):                                         # one eager warm-up step, then the capture
            m.set_input((images, valid, None, None))
            m.optimize_parameters()
        assert m._graphs["captured"]
        m.set_input((images, valid, None, None))
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert math.isfinite(float(m.mc_G_loss))
    before = {k: p.detach().clone() for k, p in m.student.named_parameters()}
    m.set_input((images, labels, None, None))
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert math.isnan(float(m.mc_G_loss)) and math.isfinite(float(m.pi_G_loss)) and math.isfinite(float(m.pa_G_loss))
    bad = [k for k, p in m.student.named_parameters() if not torch.isfinite(p).all()]
    assert not bad, bad[:5]
    assert any(not torch.equal(p.detach(), before[k]) for k, p in m.student.named_parameters())


def test_dsn_ce_error_paths(ops):
    from structure_knowledge_distillation_b200 import functions as Fn
    labels = torch.randint(0, 33, (1, 16, 16), device="cuda")
    x = torch.randn(1, 33, 4, 4, device="cuda")
    with pytest.raises(RuntimeError, match="skd_pixelwise_fwd"):
        ops.pixelwise_fwd(x, x)
    with pytest.raises(RuntimeError, match="skd_pixelwise_bwd"):
        ops.pixelwise_bwd(x, x, torch.ones((), device="cuda"))
    with pytest.raises(RuntimeError, match="skd_dsn_ce_fwd"):
        ops.dsn_ce_fwd(x, None, labels, 255, 1.0, 0.0)
    with pytest.raises(RuntimeError, match="skd_dsn_ce_fwd_train"):
        Fn.DsnCrossEntropy.apply(x.clone().requires_grad_(True), None, labels, 255, 1.0, 0.0)
    with pytest.raises(RuntimeError, match="skd_dsn_ce_bwd"):
        ops.dsn_ce_bwd(x, None, labels, 255, 1.0, 0.0, torch.ones((), device="cuda"), torch.ones((), device="cuda"))
    # the row phase keeps one row of logits and one chunk of the softmax in shared memory: 32 classes of same-size 1 024-wide logits
    # do not fit (268 KiB), and the call says so instead of launching
    x = torch.randn(1, 32, 4, 1024, device="cuda")
    lab = torch.randint(0, 32, (1, 4, 1024), device="cuda")
    with pytest.raises(RuntimeError, match="source width too large"):
        Fn.DsnCrossEntropy.apply(x.clone().requires_grad_(True), None, lab, 255, 1.0, 0.0)
    with pytest.raises(RuntimeError, match="source width too large"):
        ops.dsn_ce_bwd(x, None, lab, 255, 1.0, 0.0, torch.ones((), device="cuda"), torch.ones((), device="cuda"))
    # 19 classes at the same width fit, and are right
    x19 = torch.randn(1, 19, 4, 1024, device="cuda", dtype=torch.float64).float().double()
    rep = _dsn_check(ops, [x19], torch.randint(0, 19, (1, 4, 1024), device="cuda"), weights=(1.0, 0.0), layouts=("nhwc",))
    print("\nPARITY dsn_ce same-size 1024 wide C=19", {k: "%.2e" % v for k, v in rep.items()})


# ------------------------------------------------------------------------------------------------ pair-wise (SIMT path)
def _relu_features(g, n, c, h, w, ph, pw, quantize):
    """ReLU-like features; quantized to halves so window maxima are tied across the pooling lanes"""
    f = torch.relu(torch.randn(n, c, h, w, generator=g, device="cuda", dtype=torch.float64))
    if quantize:
        f = torch.round(f * 2) / 2
    return f.float().double()


def _zero_windows(f, ph, pw, nodes_yx, value=0):
    """every channel of the given pooling windows 0 (a student node of norm 0: rnorm = 1 / (0 + 1e-8)), or `value`"""
    for n, ny, nx in nodes_yx:
        f[n, :, ny * ph:(ny + 1) * ph, nx * pw:(nx + 1) * pw] = value


PA_CASES = [  # n, CS, CT, h, w, scale
    (2, 19, 33, 65, 129, 0.5), (2, 100, 36, 65, 129, 0.5), (2, 128, 512, 65, 129, 0.5), (3, 19, 33, 46, 61, 0.5),
    (2, 128, 512, 46, 61, 0.5), (2, 36, 20, 41, 41, 0.5), (2, 64, 128, 64, 128, 0.5), (2, 19, 33, 64, 128, 0.25),
]


@pytest.mark.parametrize("n,cs,ct,h,w,scale", PA_CASES)
def test_pairwise_simt_vs_float64(ops, n, cs, ct, h, w, scale):
    """PairWiseLoss on the SIMT path, NCHW and channels-last, ReLU features with tied maxima and all-zero student nodes: loss and
    gradient against port.pairwise_loss in float64, the gradient exactly where float64 max_pool2d's backward puts it."""
    from structure_knowledge_distillation_b200 import functions as Fn
    g = torch.Generator(device="cuda").manual_seed(h * w + cs)
    ph, pw = port.pool_patch(h, w, scale)
    nh, nw = -(-h // ph), -(-w // pw)
    assert nh * nw < Fn.PairWiseLoss.TCGEN05_MIN_NODES
    fS = _relu_features(g, n, cs, h, w, ph, pw, quantize=True)
    fT = _relu_features(g, n, ct, h, w, ph, pw, quantize=False)
    zero_nodes = [(0, 0, 0), (n - 1, nh - 1, nw - 1)]                # includes a ceil-mode edge window
    _zero_windows(fS, ph, pw, zero_nodes)
    # a zero node's gradient is scaled by 1e8 and would swamp one norm over all entries: its windows and the rest are compared apart
    in_zero = torch.zeros_like(fS, dtype=torch.bool)
    _zero_windows(in_zero, ph, pw, zero_nodes, value=True)
    Sd = fS.clone().requires_grad_(True)
    ref = port.pairwise_loss(Sd, fT, scale)
    (gref,) = torch.autograd.grad(ref, Sd)
    # yardstick for the other nodes: E = A_T - A_S is a difference of two cosines near 1 (non-negative features), so float32 Gram
    # rounding is amplified in the gradient; the same reference in float32 torch (no TF32) shows how much
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        S32 = fS.float().requires_grad_(True)
        (g32,) = torch.autograd.grad(port.pairwise_loss(S32, fT.float(), scale), S32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = saved
    e32 = _rel(g32[~in_zero], gref[~in_zero])
    worst = {}
    for lay in ("nchw", "nhwc"):
        runs = []
        for _ in range(2):
            S = _layout(fS, lay).requires_grad_(True)
            loss = Fn.PairWiseLoss.apply(S, _layout(fT, lay), ph, pw)
            (gs,) = torch.autograd.grad(loss, S)
            runs.append((loss.detach(), gs))
        assert _same_bits(runs[0][0], runs[1][0]) and _same_bits(runs[0][1], runs[1][1]), "pair-wise SIMT is not deterministic"
        loss, gs = runs[0]
        assert torch.equal(gs != 0, gref != 0), (lay, "gradient lands elsewhere than max_pool2d's backward")
        _merge(worst, dict(loss=_rel_scalar(loss, ref), grad=_rel(gs[~in_zero], gref[~in_zero]),
                           grad_zero_nodes=_rel(gs[in_zero], gref[in_zero])))
    worst["f32_grad"] = e32
    print("\nPARITY pairwise_simt", (n, cs, ct, h, w, scale), {k: "%.2e" % v for k, v in worst.items()})
    assert worst["loss"] < LOSS_TOL and worst["grad_zero_nodes"] < GRAD_TOL, worst
    assert worst["grad"] <= F32_FACTOR * e32 + GRAD_TOL, worst


@pytest.mark.parametrize("c,h,w,scale", [(128, 65, 129, 0.5), (36, 41, 41, 0.5), (20, 46, 61, 0.5), (19, 65, 129, 0.5), (33, 41, 41, 0.25)])
def test_pairwise_pool_layouts_bit_identical_and_first_max(ops, c, h, w, scale):
    """The scalar pool kernel (NCHW, or C not a multiple of 4) and the float4 NHWC kernel give the same pooled values and arg-max bit for
    bit, and the arg-max is float64 max_pool2d's: the first maximum in scan order, tied windows included."""
    g = torch.Generator(device="cuda").manual_seed(c * h + w)
    ph, pw = port.pool_patch(h, w, scale)
    f = _relu_features(g, 2, c, h, w, ph, pw, quantize=True)
    _zero_windows(f, ph, pw, [(1, 0, 1)])
    ref, idx = F.max_pool2d(f, (ph, pw), (ph, pw), 0, ceil_mode=True, return_indices=True)
    outs = {}
    for lay in ("nchw", "nhwc", "pad4"):
        pooled, arg, rnorm = ops.pairwise_pool(_layout(f, lay), ph, pw, True)
        outs[lay] = (pooled, arg, rnorm)
        assert torch.equal(pooled.double(), ref.flatten(2).transpose(1, 2)), lay
        assert torch.equal(arg.long(), idx.flatten(2).transpose(1, 2)), (lay, "arg-max is not the first maximum in scan order")
        nrm = ref.flatten(2).transpose(1, 2).pow(2).sum(2).sqrt() + 1e-8
        assert _rel(rnorm, 1.0 / nrm) < 1e-6, lay
    for lay in ("nhwc", "pad4"):
        assert all(_same_bits(a, b) for a, b in zip(outs["nchw"], outs[lay])), lay


@pytest.mark.parametrize("hw", [(31, 33), (32, 32)])
def test_pairwise_1023_and_1024_nodes(ops, hw):
    """One node below and at the switch to the wgmma path (1x1 windows): each path against float64, and the SIMT and wgmma paths on the
    same inputs within TF32 tolerance."""
    from structure_knowledge_distillation_b200 import functions as Fn
    h, w = hw
    g = torch.Generator(device="cuda").manual_seed(h * w)
    fS = _relu_features(g, 2, 64, h, w, 1, 1, quantize=False) + 0.1
    fT = _relu_features(g, 2, 128, h, w, 1, 1, quantize=False) + 0.1
    Sd = fS.clone().requires_grad_(True)
    ref = port.pairwise_loss(Sd, fT, 1.0 / min(h, w) + 1e-9)
    (gref,) = torch.autograd.grad(ref, Sd)

    def run(simt):
        old = Fn.PairWiseLoss.TCGEN05_MIN_NODES
        if simt:
            Fn.PairWiseLoss.TCGEN05_MIN_NODES = 10 ** 9
        try:
            S = _layout(fS, "nhwc").requires_grad_(True)
            loss = Fn.PairWiseLoss.apply(S, _layout(fT, "nhwc"), 1, 1)
            (gs,) = torch.autograd.grad(loss, S)
        finally:
            Fn.PairWiseLoss.TCGEN05_MIN_NODES = old
        return loss.detach(), gs

    simt, simt2 = run(True), run(True)
    assert _same_bits(simt[0], simt2[0]) and _same_bits(simt[1], simt2[1])
    default = run(False)
    rep = dict(simt_loss=_rel_scalar(simt[0], ref), simt_grad=_rel(simt[1], gref),
               default_loss=_rel_scalar(default[0], ref), default_grad=_rel(default[1], gref),
               simt_vs_default=_rel(default[1], simt[1]))
    print("\nPARITY pairwise %d nodes" % (h * w), {k: "%.2e" % v for k, v in rep.items()})
    assert rep["simt_loss"] < LOSS_TOL and rep["simt_grad"] < GRAD_TOL, rep
    if h * w < Fn.PairWiseLoss.TCGEN05_MIN_NODES:
        assert _same_bits(default[0], simt[0]) and _same_bits(default[1], simt[1])
    else:                                                              # wgmma: TF32 operands
        assert rep["default_loss"] < 1e-3 and rep["default_grad"] < 1e-2 and rep["simt_vs_default"] < 1e-2, rep
