"""MobileNetV2 student on the H100: the depthwise and BatchNorm + ReLU6 kernels against torch in float64, the 16 / 24-channel 1x1
convolutions, the network and the distillation step against tests/golden/mobilenet.pt.gz (oracle/make_golden_mobilenet.py), CUDA-graph
replay, run-to-run determinism, evaluate_main, OHEM and a two-rank step."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DW_SHAPES = [(2, 1), (1, 1), (1, 2), (1, 4)]          # (stride, dilation) of the dilated backbone's depthwise layers


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _nhwc(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("stride,dil", DW_SHAPES)
@pytest.mark.parametrize("n,c,h,w", [(2, 32, 13, 17), (2, 960, 9, 11), (1, 144, 24, 31), (2, 96, 45, 60)])
def test_depthwise_matches_float64(stride, dil, n, c, h, w):
    """Forward (with the fused BatchNorm statistics), data gradient and weight gradient against F.conv2d(groups=C) in float64; odd H
    and W, maps smaller than the dilation's reach."""
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(c + 7 * stride + dil)
    x = torch.randn(n, c, h, w, generator=g) + 0.3
    wt = torch.randn(c, 1, 3, 3, generator=g) * 0.3
    xd = x.double().requires_grad_(True); wd = wt.double().requires_grad_(True)
    ref = F.conv2d(xd, wd, stride=stride, padding=dil, dilation=dil, groups=c)
    rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
    nbt = torch.zeros((), dtype=torch.int64, device="cuda")
    y, st = ops.dwconv3x3_fwd(_nhwc(x), wt.cuda(), stride, dil, True, 0.1, rm, rv, nbt)
    y2, none = ops.dwconv3x3_fwd(_nhwc(x), wt.cuda(), stride, dil)
    assert none is None and torch.equal(y, y2)
    assert tuple(y.shape) == tuple(ref.shape)
    assert _rel(y, ref) < 1e-6
    mean, var = ref.detach().mean((0, 2, 3)), ref.detach().var((0, 2, 3), unbiased=False)
    P = ref.numel() // c
    assert _rel(st[0], mean) < 1e-6 and _rel(st[1], var) < 1e-6
    assert _rel(rm, 0.1 * mean) < 1e-6 and _rel(rv, 0.9 + 0.1 * var * P / (P - 1)) < 1e-6 and int(nbt) == 1
    dy = torch.randn(ref.shape, generator=g)
    ref.backward(dy.double())
    dx = ops.dwconv3x3_dgrad(_nhwc(dy), wt.cuda(), (n, c, h, w), stride, dil)
    dw = ops.dwconv3x3_wgrad(_nhwc(x), _nhwc(dy), stride, dil)
    assert _rel(dx, xd.grad) < 1e-6, _rel(dx, xd.grad)
    assert tuple(dw.shape) == (c, 1, 3, 3) and _rel(dw, wd.grad) < 1e-5, _rel(dw, wd.grad)
    assert torch.equal(dw, ops.dwconv3x3_wgrad(_nhwc(x), _nhwc(dy), stride, dil))


def test_depthwise_weight_gradient_long_reduction():
    """Batch 8 at 256x512, 32 channels: about 1 M pixels per channel in the weight gradient's fixed-order reduction."""
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(1)
    n, c, h, w = 8, 32, 256, 512
    x = torch.randn(n, c, h, w, generator=g)
    dy = torch.randn(n, c, h, w, generator=g)
    for stride, dil in ((1, 1), (1, 4)):
        ref = torch.nn.grad.conv2d_weight(x.cuda().double(), (c, 1, 3, 3), dy.cuda().double(), padding=dil, dilation=dil, groups=c)
        dw = ops.dwconv3x3_wgrad(_nhwc(x), _nhwc(dy), stride, dil)
        print("\nPARITY dw wgrad 8x256x512", dil, _rel(dw, ref))
        assert _rel(dw, ref) < 1e-5


def _ref_bn(x, w, b, mean, var, eps, relu6, res=None):
    z = (x - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + eps) * w[None, :, None, None] + b[None, :, None, None]
    if relu6:
        return torch.clamp(z, 0.0, 6.0)
    return z if res is None else res + z


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("mode", ["relu6", "linear", "linear_residual"])
def test_bn_act_kernels_match_torch_float64(training, mode):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(3 + training)
    n, c, h, w, eps, mom = 2, 24, 9, 13, 1e-5, 0.1
    relu6 = mode == "relu6"
    x = torch.randn(n, c, h, w, generator=g) * 2.0 + 0.5
    x[:, 5] = x[:, 5] * 0.01 + 0.3
    wt = 1 + 0.3 * torch.randn(c, generator=g); bs = 0.2 * torch.randn(c, generator=g)
    bs[3] = -100.0                                                     # channel 3: every BN output below 0
    bs[5] = 100.0                                                      # channel 5: every BN output above 6
    res = torch.randn(n, c, h, w, generator=g) if mode == "linear_residual" else None
    rm0, rv0 = 0.1 * torch.randn(c, generator=g), torch.rand(c, generator=g) + 0.5
    rm, rv, nbt = rm0.cuda(), rv0.cuda(), torch.zeros((), dtype=torch.int64, device="cuda")
    xc = _nhwc(x)
    st = ops.bnprelu_stats(xc, mom, rm, rv, nbt) if training else torch.stack([rm, rv])
    y = ops.bnact_apply(xc, st[0], st[1], wt.cuda(), bs.cuda(), eps, relu6, _nhwc(res) if res is not None else None)
    xd = x.double().requires_grad_(True)
    wd, bd = wt.double().requires_grad_(True), bs.double().requires_grad_(True)
    rd = res.double().requires_grad_(True) if res is not None else None
    if training:
        mean, var = xd.mean((0, 2, 3)), xd.var((0, 2, 3), unbiased=False)
    else:
        mean, var = rm0.double(), rv0.double()
    ref = _ref_bn(xd, wd, bd, mean, var, eps, relu6, rd)
    assert _rel(y, ref) < 1e-5
    if relu6:
        assert bool((ref[:, 3] == 0).all()) and bool((ref[:, 5] == 6).all())
    dout = torch.randn(n, c, h, w, generator=g)
    ref.backward(dout.double())
    dw, db, coef = ops.bnact_bwd_reduce(xc, _nhwc(dout), st[0], st[1], wt.cuda(), bs.cuda(), eps, relu6)
    dx = ops.bnact_bwd_dx(xc, _nhwc(dout), st[0], st[1], wt.cuda(), bs.cuda(), eps, relu6, training, coef)
    assert _rel(dx, xd.grad) < 1e-5 and _rel(dw, wd.grad) < 1e-5 and _rel(db, bd.grad) < 1e-5
    if relu6:
        assert float(dw[3]) == 0.0 and float(db[5]) == 0.0 and bool((dx[:, 3] == 0).all()) and bool((dx[:, 5] == 0).all())


@pytest.mark.parametrize("cin", [16, 24])
def test_pointwise_conv_below_one_k_chunk(cin):
    """1x1 convolutions reading 16 / 24 channels (less than one 32-channel K chunk): forward in TF32 and 3xTF32, data and weight
    gradient, against float64."""
    from structure_knowledge_distillation_b200 import functions as Fn
    g = torch.Generator().manual_seed(cin)
    x = _nhwc(torch.randn(2, cin, 23, 37, generator=g))
    wt = (torch.randn(cin * 6, cin, 1, 1, generator=g) * 0.2).cuda().contiguous(memory_format=torch.channels_last)
    ref = F.conv2d(x.double(), wt.double())
    for precise, tol in ((True, 1e-6), (False, 2e-3)):
        y = Fn.Conv2d.apply(x, wt, None, 1, 0, 1, precise)
        assert _rel(y, ref) < tol, (precise, _rel(y, ref))
    xr = x.detach().requires_grad_(True); wr = wt.detach().requires_grad_(True)
    xd = x.detach().double().requires_grad_(True); wd = wt.detach().double().requires_grad_(True)
    dy = _nhwc(torch.randn(2, cin * 6, 23, 37, generator=g))
    F.conv2d(xd, wd).backward(dy.double())
    Fn.Conv2d.apply(xr, wr, None, 1, 0, 1, True).backward(dy)
    assert _rel(xr.grad, xd.grad) < 2e-3 and _rel(wr.grad, wd.grad) < 2e-3


def _golden():
    from oracle import make_golden_mobilenet
    return make_golden_mobilenet.load()


def _student(train, batch=2):
    from oracle import cases, mobilenet_port
    from structure_knowledge_distillation_b200.networks.mobilenet import MobileNetV2
    ref = mobilenet_port.build_student(7)
    m = MobileNetV2(19).cuda()
    m.load_state_dict(ref.state_dict())
    for d, mk in zip(m.dropouts(), cases.dropout_masks(ref, batch, seed=2)):
        d.injected = mk
    return m.train(train)


def _vanishing(grads):
    """Parameters whose gradient vanishes analytically, or all but for the map border, in the fixture: a bias that reaches the loss
    only through linear layers and a train-mode BatchNorm (the projection BatchNorm's shift, which the next block's batch statistics
    remove; the DSN convolution's bias before its ABN), or through those and the zero padding of the DSN's 3x3 convolution
    (features[11..13]).  Their stored norms are cancellation residue, and no relative error of them means anything.  In the
    train-mode fixtures there are at most 17, below 2e-4 of the median norm; every other gradient is above 4e-3 of it."""
    import statistics
    med = statistics.median(v["norm"] for v in grads.values())
    skip = {k for k, v in grads.items() if v["norm"] < 1e-3 * med}
    assert len(skip) <= 17, sorted(skip)
    return skip


def _net_report(name, precise):
    from oracle import cases, make_golden_mobilenet, port
    gold = _golden()[name]
    b, h, w, train = make_golden_mobilenet.NET_CASES[name]
    m = _student(train, b)
    m.precise = precise
    images, _ = port.synthetic_batch(b, h, w, seed=11)
    out = m(images.cuda())
    loss = sum((out[i] * make_golden_mobilenet.probe(out[i].shape, 12 + i).cuda()).sum() for i in range(3))
    loss.backward()
    rep = {}
    for k, i in (("logits", 0), ("dsn", 1), ("feat", 2), ("f3", 6)):
        mine, ref = cases.at_stored(out[i].detach().contiguous(), gold[k])
        rep[k] = _rel(mine.cpu(), ref)
    rep["loss"] = abs(float(loss) - gold["loss"]) / abs(gold["loss"])
    sd = m.state_dict()
    if "running" in gold:
        rep["running"] = max(_rel(sd[k].cpu(), v) for k, v in gold["running"].items())
    worst, wn = 0.0, None
    skip = _vanishing(gold["grads"])
    for pname, p in m.named_parameters():
        gd = gold["grads"][pname]
        if pname in skip:
            continue
        e = abs(float(p.grad.double().norm()) - gd["norm"]) / max(gd["norm"], 1e-12)
        if e > worst:
            worst, wn = e, pname
    rep["worst_grad_norm"] = (worst, wn)
    return rep


@pytest.mark.parametrize("name", ["net_96x128_b2", "net_96x128_b2_eval", "net_360x480_b2"])
def test_mobilenet_forward_backward_matches_fixture(name):
    """The network (backbone convolutions in 3xTF32, the chosen mode; the head in TF32 as the ResNet18 student's) against the
    fixture; the numbers with the backbone in TF32 are printed beside it.  f3 (features[3]) is the backbone alone."""
    rep = _net_report(name, True)
    print("\nPARITY mobilenetv2 3xTF32", name, rep)
    print("PARITY mobilenetv2 TF32  ", name, _net_report(name, False))
    assert rep["f3"] < 1e-5
    assert rep["logits"] < 2e-3 and rep["dsn"] < 2e-3 and rep["feat"] < 2e-3
    assert rep.get("running", 0.0) < 5e-4 and rep["loss"] < 2e-3
    assert rep["worst_grad_norm"][0] < 5e-2, rep["worst_grad_norm"]


def _netmodel(spec, graph=False, **extra):
    from oracle import cases, espnet_port, mobilenet_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    cfg = port.StepConfig(**spec["cfg"])
    teacher, _, D = cases.build_models(seed=0, with_D=True)
    args = make_args(batch_size=spec["batch"], pi=cfg.pi, pa=cfg.pa, ho=cfg.ho, adv_loss_type=cfg.adv_type, pool_scale=cfg.pool_scale,
                     student="mobilenetv2", cuda_graph=graph, **extra)
    m = NetModel(args)
    ref = mobilenet_port.build_student(7)
    m.student.load_state_dict(ref.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for d, mk in zip(m.student.dropouts(), cases.dropout_masks(ref, spec["batch"], seed=2)):
        d.injected = mk
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    if cfg.ho and cfg.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3)).cuda()
    m.set_input((images, labels, None, None))
    return m, cfg


@pytest.mark.parametrize("name", ["step_pi_pa_360x480_b2", "step_pi_pa_ho_360x480_b2"])
def test_step_matches_fixture(name):
    from oracle import make_golden_mobilenet
    from structure_knowledge_distillation_b200.utils.criterion import CriterionDSN
    gold = _golden()[name]
    m, cfg = _netmodel(make_golden_mobilenet.STEP_CASES[name])
    assert isinstance(m.criterion, CriterionDSN)
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    assert tuple(m.preds_S[0].shape[2:]) == (45, 60) and tuple(m.preds_T[0].shape[2:]) == (45, 60)
    rep = dict(ce=m.mc_G_loss, G=m.G_loss)
    if cfg.pi: rep["pi"] = m.pi_G_loss
    if cfg.pa: rep["pa"] = m.pa_G_loss
    rep = {k: abs(float(v) - gold[k]) / abs(gold[k]) for k, v in rep.items()}
    if cfg.ho:
        m.G_solver.step()
        m.discriminator_backward()
        rep["D"] = abs(float(m.D_loss) - gold["D"]) / abs(gold["D"])
    lg = m.preds_S[0][:, :, ::4, ::4].float().cpu(); lt = m.preds_T[0][:, :, ::4, ::4].float().cpu()
    rep["logits_S_rel_l2"] = _rel(lg, gold["logits_S"]); rep["logits_T_rel_l2"] = _rel(lt, gold["logits_T"])
    worst, wn = 0.0, None
    samp_mine, samp_gold = [], []
    skip = _vanishing(gold["student_grads"])
    for pname, p in m.student.named_parameters():
        gd = gold["student_grads"].get(pname)
        if gd is None or pname in skip:
            continue
        mine = p.grad.detach().flatten().double()
        e = abs(float(mine.norm()) - gd["norm"]) / gd["norm"]
        if e > worst:
            worst, wn = e, pname
        samp_mine.append(mine[gd["idx"].to(mine.device)].cpu() / gd["norm"]); samp_gold.append(gd["samples"].double() / gd["norm"])
    sm, sg = torch.cat(samp_mine), torch.cat(samp_gold)
    rep["worst_student_grad_norm_rel"] = (worst, wn)
    rep["student_grad_samples_rel_l2"] = float((sm - sg).norm() / sg.norm())
    rep["student_grad_samples_cosine"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    print("\nPARITY mobilenetv2 step", name, rep)
    for k in ("ce", "pi", "pa", "G", "D"):
        if k in rep:
            assert rep[k] < 1e-3, (k, rep[k])
    assert rep["logits_S_rel_l2"] < 1e-3
    assert worst < 3e-2, rep["worst_student_grad_norm_rel"]
    assert rep["student_grad_samples_rel_l2"] < 3e-2 and rep["student_grad_samples_cosine"] > 0.999, rep


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + [p.detach().clone() for p in m.student.parameters()] + \
        [b.detach().clone() for b in m.student.buffers()]


def _same(a, b):
    return all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


def _state(m):
    return [{k: v.clone() for k, v in mod.state_dict().items()} for mod in (m.student, m.D_model)] + \
        [m.G_solver.flat_m.clone(), m.D_solver.flat_m.clone()]


def _rewind(m, snap):
    with torch.no_grad():
        for mod, sd in zip((m.student, m.D_model), snap[:2]):
            cur = mod.state_dict()
            for k, v in sd.items():
                cur[k].copy_(v)                                           # in place: the captured graph reads these buffers
        m.G_solver.flat_m.copy_(snap[2]); m.D_solver.flat_m.copy_(snap[3])


def test_cuda_graph_replays_equal_eager_steps_and_runs_repeat():
    """Three replays of the captured MobileNetV2 step (Pi+Pa+Ho wgan-gp, 360x480 batch 2), rewound to the starting state after the
    capture, equal three eager steps from that state bit for bit; two eager runs are bit-identical."""
    from oracle import make_golden_mobilenet
    spec = make_golden_mobilenet.STEP_CASES["step_pi_pa_ho_360x480_b2"]
    runs = []
    for _ in range(2):
        m, _ = _netmodel(spec)
        dumps = []
        for _ in range(3):
            m.optimize_parameters()
            torch.cuda.synchronize()
            dumps.append(_dump(m))
        runs.append(dumps)
        del m
    assert all(_same(a, b) for a, b in zip(runs[0], runs[1]))
    m, _ = _netmodel(spec)
    snap = _state(m)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                     # eager warm-up, capture
    assert m._graphs["captured"]
    _rewind(m, snap)
    for want in runs[0]:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), want)


def _oracle_scores(ref, image, tile, whole, scales=(1.0,), flip=False):
    """networks/evaluate.py's predict_whole / predict_multiscale / predict_sliding restated over the float64 oracle: (H, W, C) scores
    of a (1, 3, H, W) float32 CPU image (scipy's zoom for the scales, as the reference)."""
    import math
    import scipy.ndimage as nd
    _, _, H, W = image.shape
    full = torch.zeros(1, 19, H, W, dtype=torch.float64, device="cuda")

    def up(x):
        with torch.no_grad():
            return F.interpolate(ref(x)[0], size=tile, mode="bilinear", align_corners=True)
    if whole:
        hh, ww = min(tile[0], H), min(tile[1], W)
        for s in scales:
            z = torch.from_numpy(nd.zoom(image.numpy(), (1.0, 1.0, s, s), order=1, prefilter=False)).cuda().double()
            u = up(z)
            if flip:
                u = 0.5 * (u + up(z.flip(3)).flip(3))
            full[..., :hh, :ww] += u[..., :hh, :ww] / len(scales)
    else:
        img = image.cuda().double()
        stride = math.ceil(tile[0] * (1 - 1 / 3))
        rows = int(math.ceil((H - tile[0]) / stride) + 1)
        cols = int(math.ceil((W - tile[1]) / stride) + 1)
        for r in range(rows):
            for c in range(cols):
                x1, y1 = int(c * stride), int(r * stride)
                x2, y2 = min(x1 + tile[1], W), min(y1 + tile[0], H)
                x1, y1 = max(int(x2 - tile[1]), 0), max(int(y2 - tile[0]), 0)
                t = img[:, :, y1:y2, x1:x2]
                pad = torch.zeros(1, 3, tile[0], tile[1], dtype=torch.float64, device="cuda")
                pad[:, :, :t.shape[2], :t.shape[3]] = t
                full[..., y1:y2, x1:x2] += up(pad)[..., :t.shape[2], :t.shape[3]]
    return full[0].permute(1, 2, 0)


@pytest.mark.parametrize("mode", ["whole", "sliding", "multiscale_flip"])
def test_evaluate_main_matches_oracle_argmax(mode, tmp_path):
    """evaluate_main with the MobileNetV2 student (eval mode, running statistics) -- whole image, sliding padded tiles, multi-scale with
    flip -- against the float64 oracle at the same settings: the saved predictions agree except where the oracle's top-2 margin is
    below 1e-3 of its score scale."""
    import numpy as np
    from oracle import mobilenet_port
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    m = _student(False)
    ref = mobilenet_port.build_student(7).double().cuda().eval()
    whole = mode != "sliding"
    scales = (0.75, 1.0, 1.25) if mode.startswith("multiscale") else (1.0,)
    flip = mode == "multiscale_flip"
    H, W = (96, 128) if whole else (100, 161)
    g = torch.Generator().manual_seed(17)
    image = torch.randn(1, 3, H, W, generator=g) * 40.0
    label = torch.randint(0, 19, (1, H, W), generator=g)
    batches = [(image, label, [np.array([H, W, 3])], ["img0"])]
    miou, _ = evaluate_main(m, batches, 0, "64,96", 19, whole=whole, save_dir=str(tmp_path), scales=scales, flip=flip)
    pred = torch.load(tmp_path / "img0.pt").long()
    full = _oracle_scores(ref, image, (1024, 2048) if whole else (64, 96), whole, scales, flip).cpu()
    top2 = full.topk(2, dim=2).values
    near = (top2[..., 0] - top2[..., 1]) < 1e-3 * float(full.abs().max())
    want = full.argmax(2)
    bad = (pred != want) & ~near
    print("\nPARITY mobilenetv2 evaluate_main", mode, "pixels differing:", int((pred != want).sum()), "near ties:", int(near.sum()))
    assert not bool(bad.any()), int(bad.sum())
    assert 0.0 <= miou <= 1.0 and m.training is False


def test_ohem_step_runs():
    """`ohem=True` with MobileNetV2: CriterionOhemDSN on both heads, a whole NetModel step runs and keeps some but not all pixels."""
    from oracle import make_golden_mobilenet
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN
    m, _ = _netmodel(dict(make_golden_mobilenet.STEP_CASES["step_pi_pa_360x480_b2"]), ohem=True, ohem_thres=0.7, ohem_keep=20000)
    assert isinstance(m.criterion, CriterionOhemDSN)
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert float(m.G_loss) == float(m.G_loss) and 0 < float(m.criterion.last_kept) <= float((m.labels != 255).sum())
    assert all(bool(torch.isfinite(p).all()) for p in m.student.parameters())


def _ddp_worker(rank, world, port, out):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port as oport
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        torch.manual_seed(100 + rank)                                  # different init per rank: NetModel broadcasts rank 0's
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, student="mobilenetv2"))
        for d in m.student.dropouts():
            d.injected = (torch.rand(1, 128, generator=torch.Generator().manual_seed(5 + rank)) >= 0.1).float()
        p0 = m.G_solver.flat_p.clone()
        images, labels = oport.synthetic_batch(1, 360, 480, seed=7 + rank)          # each rank its own shard
        m.set_input((images, labels, None, None))
        m.G_solver._buckets = None                                                   # one exchange after backward
        m._student_phase()
        local = m.G_solver.flat_g.clone()
        m.G_solver.all_reduce_grads(world)
        summed = m.G_solver.flat_g.clone()
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        ref_sum = sum(parts)
        err = float((summed - ref_sum).norm() / ref_sum.norm())
        assert err < 1e-6, err
        lr, wd = m.G_solver.param_groups[0]["lr"], m.args.weight_decay
        m.G_solver.step()
        expect = p0 - lr * (ref_sum / world + wd * p0)                               # the mean of the per-shard gradients
        err2 = float((m.G_solver.flat_p - expect).norm() / (lr * (ref_sum / world + wd * p0)).norm())
        assert err2 < 1e-5, err2
        pg = m.G_solver.flat_p.clone()
        allp = [torch.empty_like(pg) for _ in range(world)]
        dist.all_gather(allp, pg)
        assert all(torch.equal(t, allp[0]) for t in allp), "student replicas diverged after one step"
        if rank == 0:
            out.put(("ok", err, err2))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_applies_the_mean_of_the_shard_gradients():
    """MobileNetV2 over 2 NCCL ranks: the all-reduced student gradient is the sum of the per-shard gradients and the SGD step applies
    their mean.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_ddp_worker, args=(2, 29637, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY mobilenetv2_dp_world2", res)
    assert res[0] == "ok", res
