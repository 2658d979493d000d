"""ESPNet-C student on the H100: its kernels against torch in float64, the dilated convolutions against F.conv2d, the network and the
distillation step against tests/golden/espnet.pt.gz (oracle/make_golden_espnet.py), CUDA-graph replay and run-to-run determinism."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _pitched(n, c, h, w, pitch, off, gen, scale=1.0, shift=0.0):
    """(N, C, H, W) channel slice at offset `off` of an NHWC buffer with `pitch` channels, filled with seeded values."""
    buf = (torch.randn(n, h, w, pitch, generator=gen) * scale + shift).cuda()
    return buf.permute(0, 3, 1, 2)[:, off:off + c]


def _ref_bnprelu(x, w, b, a, mean, var, eps):
    z = (x - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + eps) * w[None, :, None, None] + b[None, :, None, None]
    return torch.where(z > 0, z, a[None, :, None, None] * z)


@pytest.mark.parametrize("training", [True, False])
def test_bnprelu_kernels_match_torch_float64(training):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(0)
    n, c, h, w, eps, mom = 2, 19, 9, 13, 1e-3, 0.1
    x = _pitched(n, c, h, w, 28, 5, g, scale=2.0, shift=0.5)
    wt = (1 + 0.3 * torch.randn(c, generator=g)).cuda(); bs = (0.2 * torch.randn(c, generator=g)).cuda()
    al = (0.25 + 0.2 * torch.randn(c, generator=g)).cuda()
    bs[3] = -100.0                                                     # channel 3: every BN output negative
    rm0, rv0 = (0.1 * torch.randn(c, generator=g)).cuda(), (torch.rand(c, generator=g) + 0.5).cuda()
    rm, rv, nbt = rm0.clone(), rv0.clone(), torch.zeros((), dtype=torch.int64, device="cuda")
    if training:
        st = ops.bnprelu_stats(x, mom, rm, rv, nbt)
    else:
        st = torch.stack([rm, rv])
    y = ops.bnprelu_apply(x, st[0], st[1], wt, bs, al, eps, out_channels=20)
    xd = x.detach().double().requires_grad_(True)
    wd, bd, ad = (t.double().requires_grad_(True) for t in (wt, bs, al))
    if training:
        mean, var = xd.mean((0, 2, 3)), xd.var((0, 2, 3), unbiased=False)
        P = n * h * w
        assert _rel(st[0], mean) < 1e-6 and _rel(st[1], var) < 1e-6
        assert _rel(rm, 0.9 * rm0.double() + 0.1 * mean) < 1e-6
        assert _rel(rv, 0.9 * rv0.double() + 0.1 * var * P / (P - 1)) < 1e-6
        assert int(nbt) == 1
    else:
        mean, var = rm0.double(), rv0.double()
    ref = _ref_bnprelu(xd, wd, bd, ad, mean, var, eps)
    assert _rel(y[:, :c], ref) < 1e-5
    assert bool((y[:, c:] == 0).all())
    assert bool((ref[:, 3] <= 0).all())
    dout = _pitched(n, c, h, w, 24, 2, g)
    ref.backward(dout.double())
    dw, db, da, coef = ops.bnprelu_bwd_reduce(x, dout, st[0], st[1], wt, bs, al, eps)
    dx = ops.bnprelu_bwd_dx(x, dout, st[0], st[1], wt, bs, al, eps, training, coef, dx_channels=20)
    assert _rel(dx[:, :c], xd.grad) < 1e-5
    assert bool((dx[:, c:] == 0).all())
    assert _rel(dw, wd.grad) < 1e-5 and _rel(db, bd.grad) < 1e-5 and _rel(da, ad.grad) < 1e-5
    assert abs(float(da[3]) - float(ad.grad[3])) <= 1e-5 * abs(float(ad.grad[3]))


@pytest.mark.parametrize("n_out,add", [(64, True), (128, False), (128, True)])
def test_esp_combine_exact_and_backward(n_out, add):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(n_out + add)
    N, h, w, eps = 2, 11, 15, 1e-3
    n = n_out // 5; n1 = n_out - 4 * n
    d1 = _pitched(N, n1, h, w, ops.pad4(n1), 0, g)
    ds = [_pitched(N, n, h, w, ops.pad4(n), 0, g) for _ in range(4)]
    res = _pitched(N, n_out, h, w, n_out, 0, g) if add else None
    out = ops.empty_nhwc(N, n_out, h, w, "cuda")
    rm, rv = torch.zeros(n_out, device="cuda"), torch.ones(n_out, device="cuda")
    st = ops.esp_combine([d1] + ds, res, out, 0.1, rm, rv, None)
    a1 = ds[0]; a2 = a1 + ds[1]; a3 = a2 + ds[2]; a4 = a3 + ds[3]           # the plain-torch module's fp32 additions
    ref = torch.cat([d1, a1, a2, a3, a4], 1)
    if add:
        ref = res + ref
    assert torch.equal(out, ref)
    assert _rel(st[0], ref.double().mean((0, 2, 3))) < 1e-6 and _rel(st[1], ref.double().var((0, 2, 3), unbiased=False)) < 1e-6
    wt = (1 + 0.3 * torch.randn(n_out, generator=g)).cuda(); bs = (0.2 * torch.randn(n_out, generator=g)).cuda()
    al = (0.25 + 0.2 * torch.randn(n_out, generator=g)).cuda()
    ins = [t.detach().double().requires_grad_(True) for t in [d1] + ds + ([res] if add else [])]
    b1_, b2_, b3_, b4_ = ins[1:5]
    c = torch.cat([ins[0], b1_, b1_ + b2_, b1_ + b2_ + b3_, b1_ + b2_ + b3_ + b4_], 1)
    if add:
        c = ins[5] + c
    mean, var = c.mean((0, 2, 3)), c.var((0, 2, 3), unbiased=False)
    y = _ref_bnprelu(c, wt.double(), bs.double(), al.double(), mean, var, eps)
    dout = _pitched(N, n_out, h, w, n_out, 0, g)
    y.backward(dout.double())
    dw, db, da, coef = ops.bnprelu_bwd_reduce(out, dout, st[0], st[1], wt, bs, al, eps)
    dds, dres = ops.esp_bwd_dx(out, dout, st[0], st[1], wt, bs, al, eps, True, coef, n1, n, add)
    for got, ref_in, k in zip(dds, ins[:5], [n1] + [n] * 4):
        assert _rel(got[:, :k], ref_in.grad) < 1e-5
        assert bool((got[:, k:] == 0).all())
    if add:
        assert _rel(dres, ins[5].grad) < 1e-5


def test_input_projection_and_teacher_resample():
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(3)
    img = torch.randn(2, 3, 45, 61, generator=g).cuda()
    x4 = ops.pad_channels(img, 4)
    buf = ops.empty_nhwc(2, 20, 23, 31, "cuda")
    ops.avgpool3x3s2(x4[:, :3], buf[:, 16:19])
    ref = F.avg_pool2d(img.double(), 3, 2, 1)
    assert _rel(buf[:, 16:19], ref) < 1e-6
    buf2 = ops.empty_nhwc(2, 132, 12, 16, "cuda")
    ops.avgpool3x3s2(buf[:, 16:19], buf2[:, 128:131])
    assert _rel(buf2[:, 128:131], F.avg_pool2d(ref, 3, 2, 1)) < 1e-6
    # the teacher resample against torch's fp32 resize (what the oracle step computes); float64 only bounds both
    t = _pitched(2, 19, 46, 61, 20, 0, g)
    r = ops.resample_nhwc(t, 45, 60)
    want = F.interpolate(t.cpu().contiguous(), size=(45, 60), mode="bilinear", align_corners=True)
    assert _rel(r.cpu(), want) < 1e-6
    assert _rel(r, F.interpolate(t.double(), size=(45, 60), mode="bilinear", align_corners=True)) < 1e-5
    f = torch.randn(2, 512, 46, 61, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    want = F.interpolate(f.cpu().contiguous(), size=(45, 60), mode="bilinear", align_corners=True)
    assert _rel(ops.resample_nhwc(f, 45, 60).cpu(), want) < 1e-6


@pytest.mark.parametrize("hw,cin,cout", [((12, 16), 28, 28), ((45, 60), 28, 28), ((90, 120), 12, 12), ((7, 9), 12, 16)])
@pytest.mark.parametrize("dil", [16, 8, 2])
def test_dilated_conv_through_wgmma(hw, cin, cout, dil):
    """Dilation d with padding d on maps smaller than the padding (12x16 at 96x128 input): forward (TF32 and 3xTF32), data gradient
    and weight gradient of the ESP branches against F.conv2d in float64."""
    from structure_knowledge_distillation_b200 import functions as Fn
    g = torch.Generator().manual_seed(dil)
    h, w = hw
    x = torch.randn(2, cin, h, w, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) * 0.1).cuda().contiguous(memory_format=torch.channels_last)
    ref = F.conv2d(x.double(), wt.double(), padding=dil, dilation=dil)
    for precise, tol in ((True, 1e-5), (False, 2e-3)):
        y = Fn._esp_conv(x, Fn._esp_weight(wt, cin), 1, dil, dil, precise)
        assert _rel(y[:, :cout], ref) < tol, (precise, _rel(y[:, :cout], ref))
    xr = x.detach().requires_grad_(True); wr = wt.detach().double().requires_grad_(True)
    xd = x.detach().double().requires_grad_(True)
    dy = torch.randn(2, cout, h, w, generator=g).cuda()
    F.conv2d(xd, wr, padding=dil, dilation=dil).backward(dy.double())
    wq = wt.detach().requires_grad_(True)
    y = Fn.EspConv.apply(xr, wq, 1, dil, dil, True)
    y.backward(ops_pad(dy, y.shape[1]))
    assert _rel(xr.grad, xd.grad) < 2e-3 and _rel(wq.grad, wr.grad) < 2e-3


def ops_pad(t, c):
    from structure_knowledge_distillation_b200 import ops
    return ops.pad_channels(t, c)


def _golden():
    from oracle import make_golden_espnet
    return make_golden_espnet.load()


def _student(train):
    from oracle import espnet_port
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet_C
    ref = espnet_port.build_student(7)
    m = ESPNet_C(19).cuda()
    m.load_state_dict(ref.state_dict())
    return m.train(train)


@pytest.mark.parametrize("name", ["net_96x128_b2", "net_96x128_b2_eval", "net_360x480_b2"])
def test_espnet_forward_backward_matches_fixture(name):
    from oracle import cases, make_golden_espnet, port
    gold = _golden()[name]
    b, h, w, train = make_golden_espnet.NET_CASES[name]
    m = _student(train)
    images, _ = port.synthetic_batch(b, h, w, seed=11)
    out = m(images.cuda())
    loss = (out[0] * make_golden_espnet.probe(out[0].shape, 12).cuda()).sum() + \
        (out[2] * make_golden_espnet.probe(out[2].shape, 13).cuda()).sum()
    loss.backward()
    rep = {}
    for k, i in (("logits", 0), ("feat", 2), ("b1", 6)):
        mine, ref = cases.at_stored(out[i].detach().contiguous(), gold[k])
        rep[k] = _rel(mine.cpu(), ref)
    rep["loss"] = abs(float(loss) - gold["loss"]) / abs(gold["loss"])
    sd = m.state_dict()
    rep["running"] = max(_rel(sd[k].cpu(), v) for k, v in gold["running"].items())
    worst, wn = 0.0, None
    for pname, p in m.named_parameters():
        gd = gold["grads"][pname]
        e = abs(float(p.grad.double().norm()) - gd["norm"]) / max(gd["norm"], 1e-12)
        if e > worst:
            worst, wn = e, pname
    rep["worst_grad_norm"] = (worst, wn)
    print("\nPARITY espnet", name, rep)
    assert rep["logits"] < 1e-4 and rep["feat"] < 1e-4 and rep["b1"] < 1e-5 and rep["running"] < 1e-5
    assert rep["loss"] < 1e-4
    assert worst < 1e-2, rep["worst_grad_norm"]


def _netmodel(spec, graph=False, **extra):
    from oracle import cases, espnet_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    cfg = port.StepConfig(**spec["cfg"])
    teacher, _, D = cases.build_models(seed=0, with_D=True)
    args = make_args(batch_size=spec["batch"], pi=cfg.pi, pa=cfg.pa, ho=cfg.ho, adv_loss_type=cfg.adv_type, pool_scale=cfg.pool_scale,
                     student="espnet_c", cuda_graph=graph, **extra)
    m = NetModel(args)
    m.student.load_state_dict(espnet_port.build_student(7).state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    if cfg.ho and cfg.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3)).cuda()
    m.set_input((images, labels, None, None))
    return m, cfg


@pytest.mark.parametrize("name", ["step_pi_pa_360x480_b2", "step_pi_pa_ho_360x480_b2"])
def test_step_matches_fixture(name):
    from oracle import make_golden_espnet
    gold = _golden()[name]
    m, cfg = _netmodel(make_golden_espnet.STEP_CASES[name])
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
    samp_mine, samp_gold, worst_s, worst_s_name = [], [], 0.0, None
    for pname, p in m.student.named_parameters():
        gd = gold["student_grads"].get(pname)
        if gd is None or gd["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        e = abs(float(mine.norm()) - gd["norm"]) / gd["norm"]
        if e > worst:
            worst, wn = e, pname
        # the 16 sampled ELEMENTS of every gradient tensor: sign, direction and placement, not just magnitude
        ms, gs = mine[gd["idx"].to(mine.device)].cpu(), gd["samples"].double()
        samp_mine.append(ms / gd["norm"]); samp_gold.append(gs / gd["norm"])
        e_s = float((ms - gs).norm() / gs.norm().clamp_min(1e-30))
        if e_s > worst_s:
            worst_s, worst_s_name = e_s, pname
    sm, sg = torch.cat(samp_mine), torch.cat(samp_gold)
    rep["worst_student_grad_norm_rel"] = (worst, wn)
    rep["student_grad_samples_rel_l2"] = float((sm - sg).norm() / sg.norm())
    rep["student_grad_samples_cosine"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    rep["worst_student_grad_samples_rel_l2"] = (worst_s, worst_s_name)
    print("\nPARITY espnet step", name, rep)
    for k in ("ce", "pi", "pa", "G", "D"):
        if k in rep:
            assert rep[k] < 1e-3, (k, rep[k])
    assert worst < 3e-2, rep["worst_student_grad_norm_rel"]
    assert rep["student_grad_samples_rel_l2"] < 3e-2 and rep["student_grad_samples_cosine"] > 0.999, rep
    assert worst_s < 0.1, rep["worst_student_grad_samples_rel_l2"]


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
    """Three replays of the captured ESPNet-C step (Pi+Pa+Ho wgan-gp, 360x480 batch 2), rewound to the starting state after the
    capture, equal three eager steps from that state bit for bit; two eager runs are bit-identical."""
    from oracle import make_golden_espnet
    spec = make_golden_espnet.STEP_CASES["step_pi_pa_ho_360x480_b2"]
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


def test_eval_forward_matches_oracle_argmax():
    """The eval-mode forward (running statistics, no autograd) against the oracle in float64: the arg-max agrees except where the
    oracle's top-2 margin is below 1e-4."""
    from oracle import espnet_port
    m = _student(False)
    ref = espnet_port.build_student(7).double().eval()
    g = torch.Generator().manual_seed(5)
    img = torch.randn(1, 3, 96, 128, generator=g)
    with torch.no_grad():
        mine = m(img.cuda())[0].float().cpu()
        want = ref(img.double())[0]
    top2 = want.topk(2, dim=1).values
    ok = (mine.argmax(1) == want.argmax(1)) | ((top2[:, 0] - top2[:, 1]) < 1e-4)
    assert bool(ok.all())


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


@pytest.mark.parametrize("mode", ["whole", "sliding", "multiscale", "multiscale_flip"])
def test_evaluate_main_matches_oracle_argmax(mode, tmp_path):
    """evaluate_main with the ESPNet-C student (through model(image)[0]) -- whole image, sliding padded tiles, multi-scale, multi-scale
    with flip (batch-2 4-channel NHWC input) -- against the oracle's scores at the same settings: the saved predictions agree except
    where the oracle's top-2 margin is below 1e-4."""
    import numpy as np
    from oracle import espnet_port
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    m = _student(False)
    ref = espnet_port.build_student(7).double().cuda().eval()
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
    near = (top2[..., 0] - top2[..., 1]) < 1e-4
    want = full.argmax(2)
    bad = (pred != want) & ~near
    print("\nPARITY espnet evaluate_main", mode, "pixels differing:", int((pred != want).sum()), "near ties:", int(near.sum()))
    assert not bool(bad.any()), int(bad.sum())
    assert 0.0 <= miou <= 1.0 and m.training is False


def test_ohem_with_espnet_head_zero_only():
    """`ohem=True` with ESPNet-C: CriterionOhemDSN gets preds[1] = None and applies OHEM to head 0 alone -- equal to OhemCrossEntropy2d on
    the label-resolution logits (loss, threshold, kept count and logit gradient), and a whole NetModel step runs with it."""
    import torch.nn.functional as F
    from oracle import make_golden_espnet
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN, OhemCrossEntropy2d
    spec = dict(make_golden_espnet.STEP_CASES["step_pi_pa_360x480_b2"])
    m, _ = _netmodel(spec, ohem=True, ohem_thres=0.05, ohem_keep=20000)
    assert isinstance(m.criterion, CriterionOhemDSN)
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert float(m.G_loss) == float(m.G_loss) and 0 < float(m.criterion.last_kept) < float((m.labels != 255).sum())
    l0 = m.preds_S[0].detach().clone().requires_grad_(True)
    crit = CriterionOhemDSN(thresh=0.05, min_kept=20000)
    a = crit([l0, None], m.labels)
    a.backward()
    l1 = m.preds_S[0].detach().clone().requires_grad_(True)
    single = OhemCrossEntropy2d(255, 0.05, 20000)
    b = single(F.interpolate(l1, size=tuple(m.labels.shape[1:]), mode="bilinear", align_corners=True), m.labels)
    b.backward()
    # the fused criterion reads the low-resolution logits, the standalone one torch's upsampled copy: equal up to fp32 rounding
    ta, tb, ka, kb = float(crit.last_threshold), float(single.last_threshold), float(crit.last_kept), float(single.last_kept)
    print("\nPARITY espnet ohem", float(a), float(b), ta, tb, ka, kb, _rel(l0.grad, l1.grad))
    assert abs(float(a) - float(b)) <= 1e-4 * abs(float(b))
    assert abs(ta - tb) <= 1e-5 * abs(tb) and abs(ka - kb) <= 1e-3 * kb
    assert _rel(l0.grad, l1.grad) < 1e-3


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
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, student="espnet_c"))
        p0 = m.G_solver.flat_p.clone()
        gathered = [torch.empty_like(p0) for _ in range(world)]
        dist.all_gather(gathered, p0)
        assert all(torch.equal(t, gathered[0]) for t in gathered), "student replicas differ after construction"
        images, labels = oport.synthetic_batch(1, 360, 480, seed=7 + rank)          # each rank its own shard
        m.set_input((images, labels, None, None))
        buckets, m.G_solver._buckets = m.G_solver._buckets, None                     # first pass: one exchange after backward
        assert buckets is not None and len(buckets) >= 2
        d_state = {k: v.clone() for k, v in m.D_model.state_dict().items()}
        m._student_phase()
        local = m.G_solver.flat_g.clone()
        m.G_solver.all_reduce_grads(world)
        summed = m.G_solver.flat_g.clone()
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        ref_sum = sum(parts)
        err = float((summed - ref_sum).norm() / ref_sum.norm())
        assert err < 1e-6, err
        # second pass with the bucketed all-reduce issued from inside backward: ESPNet-C's gradients arrive through autograd's
        # post-accumulate hooks (train-mode BN: the running statistics the first pass updated do not enter the gradients)
        m.G_solver._buckets = buckets
        with torch.no_grad():
            for k, v in m.D_model.state_dict().items():
                v.copy_(d_state[k])
        m._student_phase()
        assert m._g_reduced
        torch.cuda.synchronize()
        err_o = float((m.G_solver.flat_g - summed).norm() / summed.norm())
        assert err_o < 1e-6, err_o
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
            out.put(("ok", err, err_o, err2))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_applies_the_mean_of_the_shard_gradients():
    """ESPNet-C over 2 NCCL ranks: the all-reduced student gradient is the sum of the per-shard gradients, with the plain and the
    bucketed in-backward exchange alike, and the SGD step applies their mean.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_ddp_worker, args=(2, 29617, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY espnet_dp_world2", res)
    assert res[0] == "ok", res
