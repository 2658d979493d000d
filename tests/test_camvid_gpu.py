"""CamVid on the H100: the class-weighted DSN cross entropy against float64 torch (`F.cross_entropy(..., weight=w)` per head), its
corner cases and CUDA-graph replay, the CamVid loader against a numpy restatement, 11-class distillation steps with ENet weights
against the float64 ports with torch's weighted cross entropy, and evaluate_main at 11 classes."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
C11 = 11
# the unweighted bounds of tests/test_losses_gpu.py; measured at worst on an H100: 9.1e-8 (loss) and 2.9e-6 (gradient rel-L2)
LOSS_TOL = 2e-6
GRAD_TOL = 2e-5


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().flatten().cpu(), torch.as_tensor(b).detach().double().flatten().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _rel_scalar(a, b):
    a, b = (float(x.detach()) if torch.is_tensor(x) else float(x) for x in (a, b))
    return abs(a - b) / abs(b)


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _layout(t, kind):
    t = t.float().cuda()
    if kind == "nchw":
        return t.contiguous()
    if kind == "nhwc":
        return t.contiguous(memory_format=torch.channels_last)
    n, c, h, w = t.shape                                                # pad4: a channel slice of a pitched NHWC buffer, NaN in the pad
    pitch = (c + 3) // 4 * 4 if c % 4 else c + 4
    buf = torch.full((n, h, w, pitch), float("nan"), device="cuda")
    buf[..., :c] = t.permute(0, 2, 3, 1)
    return buf.permute(0, 3, 1, 2)[:, :c]


def _weighted_ref(l64, labels, weight, ignore_index=255):
    """torch's CrossEntropyLoss(weight=w, ignore_index) of each head on the align_corners upsampled logits, 1.0 / 0.4."""
    H, W = labels.shape[1:]
    out = 0.0
    for p, wt in zip(l64, (1.0, 0.4)):
        up = F.interpolate(p, size=(H, W), mode="bilinear", align_corners=True) if p.shape[2:] != labels.shape[1:] else p
        out = out + wt * F.cross_entropy(up, labels, weight=weight, ignore_index=ignore_index)
    return out


def _kernel_paths(l64, labels, weight, layout, ignore_index=255):
    """-> eval (loss, count), training (loss, count), fused gradients of the weighted kernels."""
    from structure_knowledge_distillation_b200 import functions as Fn
    from structure_knowledge_distillation_b200 import ops
    ls = [_layout(t, layout) for t in l64]
    l1 = ls[1] if len(ls) == 2 else None
    w1 = 0.4 if len(ls) == 2 else 0.0
    ev = ops.dsn_ce_fwd(ls[0], l1, labels, ignore_index, 1.0, w1, weight)
    x = [t.detach().requires_grad_(True) for t in ls]
    tr, rows = ops.dsn_ce_fwd_train(x[0].detach(), x[1].detach() if l1 is not None else None, labels, ignore_index, 1.0, w1, weight)
    loss = Fn.DsnCrossEntropy.apply(x[0], x[1] if l1 is not None else None, labels, ignore_index, 1.0, w1, weight)
    grads = torch.autograd.grad(loss, x)
    return ev, tr, loss.detach(), grads


def _weights(g, C, zero=True):
    w = torch.rand(C, generator=g, device="cuda", dtype=torch.float64) * 5 + 0.2
    if zero and C > 2:
        w[C // 2] = 0.0                                                  # a zero-weight class
    return w


WEIGHTED_GEOMETRIES = [((45, 60), (360, 480)), ((65, 129), (512, 1024)), ((360, 480), (360, 480))]


@pytest.mark.parametrize("C", [11, 19, 21, 32])
@pytest.mark.parametrize("hw,HW", WEIGHTED_GEOMETRIES)
def test_weighted_ce_matches_float64_torch(C, hw, HW):
    g = torch.Generator(device="cuda").manual_seed(C * 1000 + HW[1])
    labels = torch.randint(0, C, (2, *HW), generator=g, device="cuda")
    labels[torch.rand(2, *HW, generator=g, device="cuda") < 0.05] = 255
    w64 = _weights(g, C)
    w32 = w64.float()
    worst = {}
    for heads, layout in ([(1, "nhwc")] if hw == HW else [(2, "nhwc"), (2, "pad4"), (1, "nchw")]):
        l64 = [(torch.randn(2, C, *hw, generator=g, device="cuda", dtype=torch.float64) * 2).float().double() for _ in range(heads)]
        xd = [t.clone().requires_grad_(True) for t in l64]
        ref = _weighted_ref(xd, labels, w32.double())
        gref = torch.autograd.grad(ref, xd)
        ev, tr, loss, grads = _kernel_paths(l64, labels, w32, layout)
        valid = labels != 255
        wsum = float(w32.double()[labels[valid]].sum())
        rep = dict(eval=_rel_scalar(ev[0], ref), train=_rel_scalar(tr[0], ref), fused_vs_unfused=_rel_scalar(ev[0], tr[0]),
                   count=abs(float(ev[1]) - wsum) / wsum, grad=max(_rel(a, b) for a, b in zip(grads, gref)))
        assert _same_bits(loss, tr[0]) and _same_bits(ev[1], tr[1]), "training forward and autograd Function differ"
        assert rep["fused_vs_unfused"] < 1e-6 and rep["count"] < 1e-6, (heads, layout, rep)
        assert rep["eval"] < LOSS_TOL and rep["train"] < LOSS_TOL and rep["grad"] < GRAD_TOL, (heads, layout, rep)
        for k, v in rep.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print("\nPARITY weighted dsn_ce C=%d %s->%s" % (C, hw, HW), {k: "%.2e" % v for k, v in worst.items()})


@pytest.mark.parametrize("C", [11, 19, 20, 32])
def test_all_ones_weights_bit_identical_to_unweighted(C):
    """Multiplying by 1.0f is exact, so all-ones weights must reproduce the unweighted loss, count and gradient bit for bit (the CT = 19
    and CT = 32 row-phase instantiations, the eval forward, one and two heads)."""
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(77 + C)
    labels = torch.randint(0, C, (2, 97, 131), generator=g, device="cuda")
    labels[torch.rand(2, 97, 131, generator=g, device="cuda") < 0.05] = 255
    ones = torch.ones(C, device="cuda")
    for heads in (2, 1):
        l = [torch.randn(2, C, 13, 17, generator=g, device="cuda").contiguous(memory_format=torch.channels_last) for _ in range(heads)]
        l1, w1 = (l[1], 0.4) if heads == 2 else (None, 0.0)
        a, b = ops.dsn_ce_fwd(l[0], l1, labels, 255, 1.0, w1), ops.dsn_ce_fwd(l[0], l1, labels, 255, 1.0, w1, ones)
        assert _same_bits(a, b), (heads, a, b)
        (a, ra), (b, rb) = ops.dsn_ce_fwd_train(l[0], l1, labels, 255, 1.0, w1), ops.dsn_ce_fwd_train(l[0], l1, labels, 255, 1.0, w1, ones)
        assert _same_bits(a, b) and _same_bits(ra, rb), heads
        go = torch.ones((), device="cuda")
        da, db = ops.dsn_ce_bwd_cols(l[0], l1, ra, 97, 1.0, w1, go, a[1]), ops.dsn_ce_bwd_cols(l[0], l1, rb, 97, 1.0, w1, go, b[1])
        assert all(_same_bits(p, q) for p, q in zip(da[:heads], db[:heads])), heads


def test_zero_weight_sum_nan_loss_zero_gradient():
    """Every present class weighted 0, and every label ignored: the loss is NaN (torch's 0/0) and the gradient exactly 0."""
    from structure_knowledge_distillation_b200.utils.criterion import CriterionCrossEntropy, CriterionDSN
    g = torch.Generator(device="cuda").manual_seed(3)
    labels = torch.randint(0, 4, (2, 97, 131), generator=g, device="cuda")
    w = [0.0] * 4 + [1.0] * 7
    for lab in (labels, torch.full_like(labels, 255)):
        for crit, heads in ((CriterionDSN(weight=w), 2), (CriterionCrossEntropy(weight=w), 1)):
            x = [torch.randn(2, C11, 13, 17, device="cuda", requires_grad=True) for _ in range(heads)]
            ref = _weighted_ref([t.detach().double() for t in x], lab, torch.tensor(w, dtype=torch.float64, device="cuda"))
            assert torch.isnan(ref)
            loss = crit(x + [None] * (2 - heads), lab)
            grads = torch.autograd.grad(loss, x)
            assert torch.isnan(loss) and all(torch.equal(gr, torch.zeros_like(gr)) for gr in grads), type(crit).__name__
            with torch.no_grad():
                assert torch.isnan(crit([t.detach() for t in x] + [None] * (2 - heads), lab))


def test_out_of_range_labels_get_weight_zero():
    """A label outside [0, C) that is not ignore_index does not index the table: it counts as a zero-weight pixel (loss, count and
    gradient equal those with that pixel ignored)."""
    g = torch.Generator(device="cuda").manual_seed(4)
    labels = torch.randint(0, C11, (2, 360, 480), generator=g, device="cuda")
    bad = torch.rand(2, 360, 480, generator=g, device="cuda") < 0.1
    labels[bad] = torch.randint(C11, 255, (int(bad.sum()),), generator=g, device="cuda")
    labels[0, 0, :7] = torch.tensor([-1, -100, 11, 12, 254, 256, 1 << 40], device="cuda")
    w = _weights(g, C11).float()
    l64 = [torch.randn(2, C11, 45, 60, generator=g, device="cuda", dtype=torch.float64).float().double() for _ in range(2)]
    clean = labels.clone()
    clean[(labels < 0) | (labels >= C11)] = 255
    ev, tr, _, grads = _kernel_paths(l64, labels, w, "nhwc")
    ev_c, tr_c, _, grads_c = _kernel_paths(l64, clean, w, "nhwc")
    assert torch.equal(ev, ev_c) and torch.equal(tr, tr_c) and all(torch.equal(a, b) for a, b in zip(grads, grads_c))
    xd = [t.clone().requires_grad_(True) for t in l64]
    ref = _weighted_ref(xd, clean, w.double())
    assert _rel_scalar(tr[0], ref) < LOSS_TOL and max(_rel(a, b) for a, b in zip(grads, torch.autograd.grad(ref, xd))) < GRAD_TOL


def test_weighted_ce_cuda_graph_replay_equals_eager():
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    labels = torch.randint(0, C11, (2, 360, 480), generator=g, device="cuda")
    w = _weights(g, C11).float()
    l0 = torch.randn(2, C11, 45, 60, generator=g, device="cuda").contiguous(memory_format=torch.channels_last)
    l1 = torch.randn(2, C11, 45, 60, generator=g, device="cuda").contiguous(memory_format=torch.channels_last)
    go = torch.ones((), device="cuda")

    def step():
        out, rows = ops.dsn_ce_fwd_train(l0, l1, labels, 255, 1.0, 0.4, w)
        return (out,) + ops.dsn_ce_bwd_cols(l0, l1, rows, 360, 1.0, 0.4, go, out[1])

    eager = [t.clone() for t in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert all(_same_bits(a, b) for a, b in zip(static, eager))


# ------------------------------------------------------------------------------------------------ the CamVid loader
def _camvid_table():
    t = np.arange(256)
    return np.where(t < C11, t, 255).astype(np.uint8)


def _camvid_getitem(image, label, crop, mean, scale, mirror):
    """CamVidDataSet.__getitem__ restated: CSDataSet's pipeline (oracle/dataset_port.cs_getitem draws the scale, crop and mirror in
    the reference's order) with the SegNet CamVid table in place of the Cityscapes id table on the label path."""
    from oracle import dataset_port as dp
    img, _, prm = dp.cs_getitem(image, label, crop, mean, scale, mirror)
    lab = _camvid_table()[label]
    if prm["scale_idx"] >= 0:
        lab = dp.resize_nearest(lab, prm["f_scale"])
    ph, pw = max(crop[0] - lab.shape[0], 0), max(crop[1] - lab.shape[1], 0)
    lab = np.pad(lab, ((0, ph), (0, pw)), constant_values=255)
    lab = lab[prm["h_off"]:prm["h_off"] + crop[0], prm["w_off"]:prm["w_off"] + crop[1]].astype(np.float32)
    return img, lab[:, ::prm["flip"]].copy()


def test_camvid_loader_matches_numpy_restatement(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset import CamVidDataSet, CSDataLoader
    (tmp_path / "train").mkdir(); (tmp_path / "trainannot").mkdir()
    rng = np.random.default_rng(6)
    sizes = [(360, 480), (360, 480), (251, 333), (407, 519)]
    raws = []
    with open(tmp_path / "train.txt", "w") as f:
        for i, (h, w) in enumerate(sizes):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            lab = rng.integers(0, 256, (h, w), dtype=np.uint8)                 # every value 0..255: classes, void and the rest
            lab[: h // 2] = rng.integers(0, 12, (h // 2, w), dtype=np.uint8)
            cv2.imwrite(str(tmp_path / "train" / ("c%d.png" % i)), img)
            cv2.imwrite(str(tmp_path / "trainannot" / ("c%d.png" % i)), lab)
            f.write("train/c%d.png trainannot/c%d.png\n" % (i, i))
            raws.append((img, lab))
    total = 0
    for crop, scale, mirror in (((360, 480), True, True), ((360, 480), False, False), ((200, 240), True, True)):
        ds = CamVidDataSet(str(tmp_path), str(tmp_path / "train.txt"), crop_size=crop, scale=scale, mirror=mirror)
        random.seed(8); np.random.seed(8)
        batches = list(CSDataLoader(ds, batch_size=1))
        random.seed(8); np.random.seed(8)
        for k, (images, labels, size, name) in enumerate(batches):
            wi, wl = _camvid_getitem(raws[k][0], raws[k][1], crop, (128, 128, 128), scale, mirror)
            assert images.is_cuda and labels.dtype == torch.int64 and name == ["c%d" % k]
            assert np.array_equal(images[0].cpu().numpy(), wi), (crop, k)
            assert np.array_equal(labels[0].cpu().numpy().astype(np.float32), wl), (crop, k)
            assert set(np.unique(wl)) <= set(range(C11)) | {255.0}
            total += 1
    print("\nPARITY camvid loader %d samples bit-exact vs the numpy restatement" % total)


# ------------------------------------------------------------------------------------------------ 11-class steps with ENet weights
def _skewed_labels(batch, h, w, seed):
    """CamVid-like imbalance: class k drawn with probability ~ (k + 1)^-2, 5 % ignored."""
    g = torch.Generator().manual_seed(seed)
    p = 1.0 / torch.arange(1, C11 + 1, dtype=torch.float64) ** 2
    labels = torch.multinomial(p / p.sum(), batch * h * w, replacement=True, generator=g).view(batch, h, w)
    labels[torch.rand(batch, h, w, generator=g) < 0.05] = 255
    return labels


def _enet_weights(labels, c=1.02):
    valid = labels[labels != 255]
    p = torch.bincount(valid, minlength=C11).double() / valid.numel()
    return (1.0 / torch.log(c + p)).float()


def _netmodel(student, batch, h, w, cfg, graph=False, **extra):
    from oracle import cases, espnet_full_port, espnet_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    teacher, s_port, D = cases.build_models(seed=0, with_D=True, classes=C11)
    if student == "espnet_c":
        s_port = espnet_port.build_student(7, classes=C11)
    elif student == "espnet":
        s_port = espnet_full_port.build_student(7, classes=C11)
    images, _ = port.synthetic_batch(batch, h, w, seed=1, classes=C11)
    labels = _skewed_labels(batch, h, w, seed=2)
    weights = _enet_weights(labels)
    args = make_args(classes_num=C11, batch_size=batch, pi=cfg.pi, pa=cfg.pa, ho=cfg.ho, adv_loss_type=cfg.adv_type,
                     pool_scale=cfg.pool_scale, student=student, cuda_graph=graph, class_weights=weights.tolist(), **extra)
    m = NetModel(args)
    m.student.load_state_dict(s_port.state_dict()); m.teacher.load_state_dict(teacher.state_dict()); m.D_model.load_state_dict(D.state_dict())
    masks = cases.dropout_masks(s_port, batch, seed=2) if student == "resnet18" else []
    for drop, mk in zip(m.student.dropouts(), masks):
        drop.injected = mk
    if cfg.ho and cfg.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    m.set_input((images, labels, None, None))
    return m, dict(teacher=teacher, student=s_port, D=D, images=images, labels=labels, masks=masks, weights=weights)


def _grad_report(m, grads):
    worst, sm, sg = 0.0, [], []
    for pname, p in m.student.named_parameters():
        gd = grads.get(pname)
        if gd is None or gd["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        worst = max(worst, abs(float(mine.norm()) - gd["norm"]) / gd["norm"])
        sm.append(mine[gd["idx"].to(mine.device)].cpu() / gd["norm"]); sg.append(gd["samples"].double().cpu() / gd["norm"])
    sm, sg = torch.cat(sm), torch.cat(sg)
    return worst, float((sm - sg).norm() / sg.norm()), float((sm * sg).sum() / (sm.norm() * sg.norm()))


@pytest.mark.parametrize("student", ["resnet18", "espnet_c", "espnet"])
def test_11_class_weighted_step_matches_float64_port(student, monkeypatch):
    """Pi + Pa + Ho wgan-gp at 11 classes, batch 2 at 360 x 480, with ENet class weights: NetModel against the students' float64 ports
    whose task loss is torch's weighted cross entropy (CrossEntropyLoss(weight=w) in place of the unweighted one)."""
    from oracle import cases, espnet_full_port, espnet_port, port
    from structure_knowledge_distillation_b200.networks.pspnet_combine import Conv2d
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    m, ref = _netmodel(student, 2, 360, 480, cfg)
    for mod in m.student.modules():                                    # 3xTF32 student forward, as the 21-class port test
        if isinstance(mod, Conv2d):
            mod.precise = True
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    assert m.preds_S[0].shape[1] == C11 and m.criterion.weight.is_cuda
    T, S = ref["teacher"].cuda().double(), ref["student"].cuda().double()
    for drop, mk in zip(S.dropouts() if student == "resnet18" else [], ref["masks"]):
        drop.injected = mk.cuda().double()
    D = espnet_port.size_aware_D(ref["D"], tuple(m._d_inputs()[0].shape[2:])).cuda().double()
    w64 = ref["weights"].double().cuda()
    ce = F.cross_entropy
    monkeypatch.setattr(F, "cross_entropy", lambda inp, tgt, **kw: ce(inp, tgt, weight=w64, **kw))
    step = {"resnet18": port.distill_step, "espnet_c": espnet_port.distill_step, "espnet": espnet_full_port.distill_step}[student]
    out = step(T, S, D, ref["images"].cuda().double(), ref["labels"].cuda(), cfg, gp_alpha=m.criterion_AdditionalGP.alpha.double())
    monkeypatch.undo()
    rep = {k: abs(float(v) - out[k]) / abs(out[k]) for k, v in dict(ce=m.mc_G_loss, pi=m.pi_G_loss, pa=m.pa_G_loss, G=m.G_loss).items()}
    heads = 2 if student == "resnet18" else 1
    unweighted = _weighted_ref([p.detach() for p in out["preds_S"][:heads]], ref["labels"].cuda(), None)
    unweighted_ce_gap = abs(float(m.mc_G_loss) - float(unweighted))
    grads = cases.grad_digest(S.named_parameters())
    rep["worst_student_grad_norm_rel"], rep["student_grad_samples_rel_l2"], rep["student_grad_samples_cosine"] = _grad_report(m, grads)
    print("\nPARITY camvid weighted step vs port", student, rep, "weighted - unweighted CE: %.3f" % unweighted_ce_gap)
    assert unweighted_ce_gap > 1e-2                                    # the weights change the loss the test compares
    for k in ("ce", "pi", "pa", "G"):
        assert rep[k] < 1e-3, (k, rep[k])
    assert rep["worst_student_grad_norm_rel"] < 2e-2 and rep["student_grad_samples_rel_l2"] < 2e-2, rep
    assert rep["student_grad_samples_cosine"] > 0.999, rep


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + [p.detach().clone() for p in m.student.parameters()] + \
        [b.detach().clone() for b in m.student.buffers()] + [p.detach().clone() for p in m.D_model.parameters()]


@pytest.mark.parametrize("student", ["resnet18", "espnet"])
def test_11_class_weighted_cuda_graph_replays_equal_eager_steps(student):
    from oracle import port
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    m, _ = _netmodel(student, 2, 360, 480, cfg)
    eager = []
    for _ in range(2):
        m.optimize_parameters(); torch.cuda.synchronize(); eager.append(_dump(m))
    del m
    m, _ = _netmodel(student, 2, 360, 480, cfg)
    snap = [{k: v.clone() for k, v in mod.state_dict().items()} for mod in (m.student, m.D_model)] + \
        [m.G_solver.flat_m.clone(), m.D_solver.flat_m.clone()]
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()
    assert m._graphs["captured"]
    with torch.no_grad():
        for mod, sd in zip((m.student, m.D_model), snap[:2]):
            cur = mod.state_dict()
            for k, v in sd.items():
                cur[k].copy_(v)
        m.G_solver.flat_m.copy_(snap[2]); m.D_solver.flat_m.copy_(snap[3])
    for want in eager:
        m.optimize_parameters(); torch.cuda.synchronize()
        got = _dump(m)
        assert all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(got, want))


@pytest.mark.parametrize("kind", ["resnet18", "espnet_c"])
def test_seg_model_weighted_step(kind):
    """SegModel passes args.class_weights to its task loss: its step's loss is the weighted loss of its own logits."""
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    labels = _skewed_labels(2, 360, 480, seed=9)
    w = _enet_weights(labels)
    m = SegModel(make_args(batch_size=2, classes_num=C11, seg_model=kind, class_weights=w))
    assert torch.equal(m.criterion.weight, w.cuda())
    m.set_input((torch.randn(2, 3, 360, 480), labels, None, None))
    m.optimize_parameters(); torch.cuda.synchronize()
    heads = 2 if kind == "resnet18" else 1
    ref = _weighted_ref([p.detach().double() for p in m.preds[:heads]], labels.cuda(), w.double().cuda())
    assert _rel_scalar(m.mc_G_loss, ref) < 1e-5, (float(m.mc_G_loss), float(ref))


# ------------------------------------------------------------------------------------------------ evaluation at 11 classes
def test_evaluate_main_11_classes_one_tile(tmp_path):
    """evaluate_main(model, CSDataLoader(CamVidDataSet(..., (360, 480), scale=False, mirror=False)), '0', '360,480', 11, whole=False):
    one sliding tile (one forward) per 360 x 480 image, and the IU array of the confusion matrix that a numpy restatement builds
    from the saved predictions and the raw label files through the CamVid table."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset import CamVidDataSet, CSDataLoader
    from structure_knowledge_distillation_b200.networks import evaluate as E
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet_C
    torch.manual_seed(1)
    m = ESPNet_C(C11).cuda().eval()
    calls = []
    m.register_forward_hook(lambda mod, inp, out: calls.append(tuple(inp[0].shape)))
    (tmp_path / "val").mkdir(); (tmp_path / "valannot").mkdir()
    rng = np.random.default_rng(12)
    raw_labels = []
    with open(tmp_path / "val.txt", "w") as f:
        for i in range(3):
            cv2.imwrite(str(tmp_path / "val" / ("v%d.png" % i)), rng.integers(0, 256, (360, 480, 3), dtype=np.uint8))
            lab = rng.integers(0, 12, (360, 480), dtype=np.uint8); lab[:, :9] = 200
            cv2.imwrite(str(tmp_path / "valannot" / ("v%d.png" % i)), lab)
            f.write("val/v%d.png valannot/v%d.png\n" % (i, i))
            raw_labels.append(lab)
    ds = CamVidDataSet(str(tmp_path), str(tmp_path / "val.txt"), crop_size=(360, 480), scale=False, mirror=False)
    miou, ious = E.evaluate_main(m, CSDataLoader(ds, batch_size=1), "0", "360,480", C11, whole=False, save_dir=str(tmp_path / "pt"))
    assert calls == [(1, 3, 360, 480)] * 3
    conf = np.zeros((C11, C11), np.int64)
    for i, lab in enumerate(raw_labels):
        pred = torch.load(tmp_path / "pt" / ("v%d.pt" % i)).long().numpy()
        assert pred.shape == (360, 480) and pred.max() < C11
        gt = _camvid_table()[lab].astype(np.int64)
        keep = gt != 255
        conf += np.bincount(gt[keep] * C11 + pred[keep], minlength=C11 * C11).reshape(C11, C11)
    tp = np.diag(conf)
    want = tp / np.maximum(1.0, conf.sum(1) + conf.sum(0) - tp)
    print("\nPARITY camvid evaluate_main mean IU %.6f" % miou)
    assert len(ious) == C11 and np.array_equal(ious, want) and miou == want.mean()
