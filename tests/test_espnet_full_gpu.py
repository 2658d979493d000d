"""Full ESPNet student on the H100: the transposed convolution, plain BatchNorm and resize-adjoint kernels against torch in float64,
the network and the distillation step against tests/golden/espnet_full.pt.gz (oracle/make_golden_espnet_full.py), CUDA-graph replay,
evaluation, OHEM and the two-rank step."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("cin,cout,h,w", [(19, 19, 45, 60), (19, 19, 90, 120), (7, 5, 13, 17)])
def test_transposed_conv_forward_dgrad_wgrad_float64(cin, cout, h, w):
    from structure_knowledge_distillation_b200 import functions as Fn, ops
    g = torch.Generator().manual_seed(cin * h)
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(cin, cout, 2, 2, generator=g) * 0.3
    dy = torch.randn(2, cout, 2 * h, 2 * w, generator=g)
    xd, wd = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    ref = F.conv_transpose2d(xd, wd, stride=2)
    ref.backward(dy.double())
    xp = ops.pad_channels(x.cuda(), ops.pad4(cin)).requires_grad_(True)
    wq = wt.cuda().requires_grad_(True)
    y = Fn.EspConvTranspose.apply(xp, wq)
    assert tuple(y.shape) == (2, ops.pad4(cout), 2 * h, 2 * w) and bool((y[:, cout:] == 0).all())
    assert _rel(y[:, :cout], ref) < 1e-6                                             # 3xTF32
    y.backward(ops.pad_channels(dy.cuda(), ops.pad4(cout)))
    assert _rel(xp.grad[:, :cin], xd.grad) < 2e-3 and _rel(wq.grad, wd.grad) < 2e-3   # TF32, as every ESPNet data / weight gradient
    print("\nPARITY convT", cin, cout, h, w, _rel(y[:, :cout], ref), _rel(xp.grad[:, :cin], xd.grad), _rel(wq.grad, wd.grad))


@pytest.mark.parametrize("training", [True, False])
def test_batchnorm_without_prelu_float64(training):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(2)
    n, c, h, w, eps, mom = 2, 19, 9, 13, 1e-3, 0.1
    x = (torch.randn(n, h, w, 20, generator=g) * 2 + 0.5).cuda().permute(0, 3, 1, 2)[:, :c]
    wt = (1 + 0.3 * torch.randn(c, generator=g)).cuda(); bs = (0.2 * torch.randn(c, generator=g)).cuda()
    rm, rv = (0.1 * torch.randn(c, generator=g)).cuda(), (torch.rand(c, generator=g) + 0.5).cuda()
    st = ops.bnprelu_stats(x, mom, rm.clone(), rv.clone(), None) if training else torch.stack([rm, rv])
    y = ops.bnprelu_apply(x, st[0], st[1], wt, bs, None, eps, out_channels=20)
    xd = x.detach().double().requires_grad_(True)
    wd, bd = wt.double().requires_grad_(True), bs.double().requires_grad_(True)
    mean, var = (xd.mean((0, 2, 3)), xd.var((0, 2, 3), unbiased=False)) if training else (rm.double(), rv.double())
    ref = (xd - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + eps) * wd[None, :, None, None] + bd[None, :, None, None]
    assert _rel(y[:, :c], ref) < 1e-5 and bool((y[:, c:] == 0).all())
    assert bool((ref < 0).any())                                                     # negative outputs pass unchanged (no PReLU)
    dout = torch.randn(n, c, h, w, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    ref.backward(dout.double())
    dw, db, da, coef = ops.bnprelu_bwd_reduce(x, dout, st[0], st[1], wt, bs, None, eps)
    dx = ops.bnprelu_bwd_dx(x, dout, st[0], st[1], wt, bs, None, eps, training, coef, dx_channels=20)
    assert da is None
    assert _rel(dx[:, :c], xd.grad) < 1e-5 and _rel(dw, wd.grad) < 1e-5 and _rel(db, bd.grad) < 1e-5


@pytest.mark.parametrize("src,dst", [((360, 480), (46, 61)), ((96, 128), (13, 17)), ((512, 1024), (65, 129))])
def test_resize_adjoint_float64_and_bit_identical(src, dst):
    from structure_knowledge_distillation_b200 import functions as Fn
    g = torch.Generator().manual_seed(4)
    t = torch.randn(2, 19, *src, generator=g)
    dout = torch.randn(2, 19, *dst, generator=g)
    td = t.double().requires_grad_(True)
    F.interpolate(td, size=dst, mode="bilinear", align_corners=True).backward(dout.double())
    grads = []
    for _ in range(2):
        tc = t.cuda().requires_grad_(True)
        y = Fn.ResampleBilinear.apply(tc, *dst)
        assert _rel(y, F.interpolate(t, size=dst, mode="bilinear", align_corners=True)) < 1e-6      # torch's fp32 resize
        y.backward(dout.cuda())
        grads.append(tc.grad.clone())
    print("\nPARITY resize adjoint", src, dst, _rel(grads[0], td.grad))
    assert _rel(grads[0], td.grad) < 1e-4          # float32 source coordinates, as the forward (about 2e-5 at 360 -> 46 rows)
    assert torch.equal(grads[0], grads[1])


def test_cross_entropy_on_full_resolution_logits_is_exact():
    """CriterionCrossEntropy on logits at the label size: the upsample is the identity, the loss is F.cross_entropy's."""
    from structure_knowledge_distillation_b200.utils.criterion import CriterionCrossEntropy
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(2, 19, 64, 96, generator=g).cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    labels = torch.randint(0, 19, (2, 64, 96), generator=g).cuda()
    labels[:, :5] = 255
    loss = CriterionCrossEntropy()([logits, None], labels)
    loss.backward()
    ld = logits.detach().double().requires_grad_(True)
    ref = F.cross_entropy(ld, labels, ignore_index=255)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-6 * abs(float(ref))
    assert _rel(logits.grad, ld.grad) < 1e-5


def _golden():
    from oracle import make_golden_espnet_full
    return make_golden_espnet_full.load()


def _student(train):
    from oracle import espnet_full_port
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet
    m = ESPNet(19).cuda()
    m.load_state_dict(espnet_full_port.build_student(7).state_dict())
    return m.train(train)


@pytest.mark.parametrize("name", ["net_96x128_b2", "net_96x128_b2_eval", "net_360x480_b2"])
def test_espnet_forward_backward_matches_fixture(name):
    from oracle import cases, make_golden_espnet, make_golden_espnet_full, port
    gold = _golden()[name]
    b, h, w, train = make_golden_espnet_full.NET_CASES[name]
    m = _student(train)
    images, _ = port.synthetic_batch(b, h, w, seed=11)
    out = m(images.cuda())
    assert tuple(out[0].shape) == (b, 19, h, w)
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
    print("\nPARITY espnet_full", name, rep)
    assert rep["logits"] < 1e-3 and rep["feat"] < 1e-4 and rep["b1"] < 1e-5 and rep["running"] < 1e-4
    assert rep["loss"] < 1e-3
    assert worst < 1e-2, rep["worst_grad_norm"]


def _netmodel(spec, graph=False, **extra):
    from oracle import cases, espnet_full_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    cfg = port.StepConfig(**spec["cfg"])
    teacher, _, D = cases.build_models(seed=0, with_D=True)
    args = make_args(batch_size=spec["batch"], pi=cfg.pi, pa=cfg.pa, ho=cfg.ho, adv_loss_type=cfg.adv_type, pool_scale=cfg.pool_scale,
                     student="espnet", cuda_graph=graph, **extra)
    m = NetModel(args)
    m.student.load_state_dict(espnet_full_port.build_student(7).state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    if cfg.ho and cfg.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3)).cuda()
    m.set_input((images, labels, None, None))
    return m, cfg


@pytest.mark.parametrize("name", ["step_pi_pa_360x480_b2", "step_pi_pa_ho_360x480_b2"])
def test_step_matches_fixture(name):
    from oracle import make_golden_espnet_full
    gold = _golden()[name]
    m, cfg = _netmodel(make_golden_espnet_full.STEP_CASES[name])
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    assert tuple(m.preds_S[0].shape[2:]) == (360, 480) and tuple(m.preds_T[0].shape[2:]) == (360, 480)
    assert tuple(m.preds_T[-5].shape[2:]) == (45, 60) and tuple(m.logits_T.shape[2:]) == (46, 61)
    rep = dict(ce=m.mc_G_loss, G=m.G_loss)
    if cfg.pi: rep["pi"] = m.pi_G_loss
    if cfg.pa: rep["pa"] = m.pa_G_loss
    rep = {k: abs(float(v) - gold[k]) / abs(gold[k]) for k, v in rep.items()}
    if cfg.ho:
        m.G_solver.step()
        m.discriminator_backward()
        rep["D"] = abs(float(m.D_loss) - gold["D"]) / abs(gold["D"])
    lg = m.preds_S[0][:, :, ::16, ::16].float().cpu(); lt = m.preds_T[0][:, :, ::16, ::16].float().cpu()
    rep["logits_S_rel_l2"] = _rel(lg, gold["logits_S"]); rep["logits_T_rel_l2"] = _rel(lt, gold["logits_T"])
    worst, wn = 0.0, None
    samp_mine, samp_gold = [], []
    for pname, p in m.student.named_parameters():
        gd = gold["student_grads"].get(pname)
        if gd is None or gd["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        e = abs(float(mine.norm()) - gd["norm"]) / gd["norm"]
        if e > worst:
            worst, wn = e, pname
        samp_mine.append(mine[gd["idx"].to(mine.device)].cpu() / gd["norm"]); samp_gold.append(gd["samples"].double() / gd["norm"])
    sm, sg = torch.cat(samp_mine), torch.cat(samp_gold)
    rep["worst_student_grad_norm_rel"] = (worst, wn)
    rep["student_grad_samples_rel_l2"] = float((sm - sg).norm() / sg.norm())
    print("\nPARITY espnet_full step", name, rep)
    for k in ("ce", "pi", "pa", "G", "D"):
        if k in rep:
            assert rep[k] < 1e-3, (k, rep[k])
    assert rep["logits_S_rel_l2"] < 1e-3 and rep["logits_T_rel_l2"] < 1e-3, rep
    assert worst < 3e-2, rep["worst_student_grad_norm_rel"]
    assert rep["student_grad_samples_rel_l2"] < 3e-2, rep


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + [p.detach().clone() for p in m.student.parameters()] + \
        [b.detach().clone() for b in m.student.buffers()]


def _same(a, b):
    return all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


def test_cuda_graph_replays_equal_eager_steps():
    """Two replays of the captured full-ESPNet step (Pi+Pa+Ho wgan-gp, 360x480 batch 2), rewound to the starting state, equal two eager
    steps bit for bit; two eager runs are bit-identical (the resize adjoint is a fixed-order gather)."""
    from oracle import make_golden_espnet_full
    spec = make_golden_espnet_full.STEP_CASES["step_pi_pa_ho_360x480_b2"]
    runs = []
    for _ in range(2):
        m, _ = _netmodel(spec)
        dumps = []
        for _ in range(2):
            m.optimize_parameters()
            torch.cuda.synchronize()
            dumps.append(_dump(m))
        runs.append(dumps)
        del m
    assert all(_same(a, b) for a, b in zip(runs[0], runs[1]))
    m, _ = _netmodel(spec)
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
    for want in runs[0]:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), want)


@pytest.mark.parametrize("mode", ["whole", "sliding", "multiscale_flip"])
def test_evaluate_main_matches_oracle_argmax(mode, tmp_path):
    import numpy as np
    from oracle import espnet_full_port
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    from test_espnet_gpu import _oracle_scores
    m = _student(False)
    ref = espnet_full_port.build_student(7).double().cuda().eval()
    whole = mode != "sliding"
    scales = (0.75, 1.0, 1.25) if mode.startswith("multiscale") else (1.0,)
    flip = mode == "multiscale_flip"
    H, W = (96, 128) if whole else (100, 161)
    g = torch.Generator().manual_seed(17)
    image = torch.randn(1, 3, H, W, generator=g) * 40.0
    label = torch.randint(0, 19, (1, H, W), generator=g)
    miou, _ = evaluate_main(m, [(image, label, [np.array([H, W, 3])], ["img0"])], 0, "64,96", 19, whole=whole, save_dir=str(tmp_path),
                            scales=scales, flip=flip)
    pred = torch.load(tmp_path / "img0.pt").long()
    full = _oracle_scores(ref, image, (1024, 2048) if whole else (64, 96), whole, scales, flip).cpu()
    top2 = full.topk(2, dim=2).values
    near = (top2[..., 0] - top2[..., 1]) < 1e-4
    bad = (pred != full.argmax(2)) & ~near
    print("\nPARITY espnet_full evaluate_main", mode, "pixels differing:", int((pred != full.argmax(2)).sum()), "near ties:", int(near.sum()))
    assert not bool(bad.any()), int(bad.sum())
    assert 0.0 <= miou <= 1.0 and m.training is False


def test_ohem_step_head_zero():
    from oracle import make_golden_espnet_full
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN, OhemCrossEntropy2d
    m, _ = _netmodel(make_golden_espnet_full.STEP_CASES["step_pi_pa_360x480_b2"], ohem=True, ohem_thres=0.05, ohem_keep=20000)
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
    b = single(l1, m.labels)                                                 # full-resolution logits: no upsample
    b.backward()
    print("\nPARITY espnet_full ohem", float(a), float(b), float(crit.last_kept), float(single.last_kept), _rel(l0.grad, l1.grad))
    assert abs(float(a) - float(b)) <= 1e-5 * abs(float(b))
    assert float(crit.last_kept) == float(single.last_kept)
    assert _rel(l0.grad, l1.grad) < 1e-5


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
        torch.manual_seed(100 + rank)
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, student="espnet"))
        p0 = m.G_solver.flat_p.clone()
        images, labels = oport.synthetic_batch(1, 360, 480, seed=7 + rank)
        m.set_input((images, labels, None, None))
        m.G_solver._buckets = None
        m._student_phase()
        local = m.G_solver.flat_g.clone()
        m.G_solver.all_reduce_grads(world)
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        ref_sum = sum(parts)
        err = float((m.G_solver.flat_g - ref_sum).norm() / ref_sum.norm())
        assert err < 1e-6, err
        lr, wd = m.G_solver.param_groups[0]["lr"], m.args.weight_decay
        m.G_solver.step()
        expect = p0 - lr * (ref_sum / world + wd * p0)
        err2 = float((m.G_solver.flat_p - expect).norm() / (lr * (ref_sum / world + wd * p0)).norm())
        assert err2 < 1e-5, err2
        if rank == 0:
            out.put(("ok", err, err2))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_applies_the_mean_of_the_shard_gradients():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29619, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY espnet_full_dp_world2", res)
    assert res[0] == "ok", res
