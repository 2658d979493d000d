"""SegModel on the H100: two training steps of PSPNet-ResNet101 (19 / 21 classes, CriterionDSN / CriterionOhemDSN) and of the ResNet18-PSP
baseline against the reference's steps (tests/golden/seg_steps.pt.gz, oracle/make_golden_seg.py), the split-precision policies, CUDA-graph
replay, every network kind, the launch list, the checkpoint round trip into NetModel's teacher, the full-size step's peak memory and two
ranks."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# DESIGN.md §4 "The teacher in training": measured on an H100 80GB HBM3 (700 W) with the default policies, the first step: logits
# <= 2.4e-3 rel-L2, worst gradient norm 2.7e-2, sampled gradients 5.4e-2, update 6.0e-2; the bounds leave about 2-3x headroom.
TOL = dict(loss=1e-3, logits=5e-3, grad_norm=8e-2, grad_samples=0.15, update=0.15)
# OHEM's second step: which pixels are kept is decided by comparing probabilities with a threshold, so the first step's TF32 gradient
# difference moves pixels in or out of the kept set (measured 4.8e-3)
OHEM_STEP2_LOSS = 1e-2


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def _golden():
    from oracle import make_golden_seg
    return make_golden_seg.load()


def _seg(name, policy=None, graph=False, **extra):
    """SegModel of a golden case with the case's weights, dropout masks and batch."""
    from oracle import make_golden_seg as G
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    arch, classes, ohem = G.CASES[name]
    kw = dict(batch_size=G.BATCH, classes_num=classes, seg_model=arch, lr_g=G.LR, momentum=G.MOMENTUM, weight_decay=G.WEIGHT_DECAY,
              ohem=ohem, ohem_thres=G.OHEM_THRES, ohem_keep=G.OHEM_KEEP, cuda_graph=graph)
    if policy is not None:
        kw["seg_precision"] = policy
    kw.update(extra)
    m = SegModel(make_args(**kw))
    src = G.build_net(arch, classes)
    m.model.load_state_dict(src.state_dict())
    for d, mk in zip(m.model.dropouts(), G.masks(src)):
        d.injected = mk
    m.set_input(G.batch(classes))
    return m, src


def _vanishing(grads):
    """Gradients that vanish analytically in train mode (a bias followed by a batch-statistics BN: the DSN convolution's bias), whose
    stored norms are cancellation residue."""
    import statistics
    med = statistics.median(v["norm"] for v in grads.values())
    return {k for k, v in grads.items() if v["norm"] < 1e-3 * med}


def _report(name, policy=None):
    """Two steps against the golden -> per-step errors: loss, logits, worst per-tensor gradient norm, sampled gradients (rel-L2 of the
    samples scaled by their tensor's norm) and the SGD update at the sampled positions."""
    from oracle import make_golden_seg as G
    gold = _golden()[name]
    m, src = _seg(name, policy)
    p0 = {k: v.detach().flatten()[G.strided(v.numel())].clone() for k, v in src.named_parameters()}
    reps = []
    for gs in gold["steps"]:
        m.forward(); m.G_solver.zero_grad(); m.backward()
        rep = dict(loss=abs(float(m.G_loss) - gs["loss"]) / abs(gs["loss"]), logits=_rel(m.preds[0].detach().contiguous(), gs["logits"]),
                   grad_norm=(0.0, None))
        skip = _vanishing(gs["grads"])
        sm, sg = [], []
        for pname, p in m.model.named_parameters():
            gd = gs["grads"][pname]
            if pname in skip:
                continue
            g = p.grad.detach().flatten().double()
            e = abs(float(g.norm()) - gd["norm"]) / gd["norm"]
            if e > rep["grad_norm"][0]:
                rep["grad_norm"] = (e, pname)
            sm.append(g[gd["idx"].to(g.device)].cpu() / gd["norm"]); sg.append(gd["samples"].double() / gd["norm"])
        rep["grad_samples"] = _rel(torch.cat(sm), torch.cat(sg))
        m._update()
        um, ug = [], []
        for pname, p in m.model.named_parameters():
            if pname in skip:
                continue
            pm = p.detach().flatten()[G.strided(p.numel()).to(p.device)].cpu()
            um.append(pm - p0[pname]); ug.append(gs["params"][pname] - p0[pname])
        rep["update"] = _rel(torch.cat(um), torch.cat(ug))
        reps.append(rep)
    return reps


# ---- kernel passes at the shapes only the ResNet101 training step reaches, against float64 -------------------------------------------
# (name, N, Cin, Cout, H, W, k, stride, pad, bias): batch 1 at the 512x1024 crop's feature sizes
CONV_SHAPES = [
    ("bottleneck_1x1_256_to_1024", 1, 256, 1024, 65, 129, 1, 1, 0, False),
    ("bottleneck_1x1_1024_to_256", 1, 1024, 256, 65, 129, 1, 1, 0, False),
    ("bottleneck_1x1_512_to_2048", 1, 512, 2048, 65, 129, 1, 1, 0, False),
    ("bottleneck_1x1_2048_to_512", 1, 2048, 512, 65, 129, 1, 1, 0, False),
    ("layer2_downsample_1x1_s2_256_to_512", 1, 256, 512, 129, 257, 1, 2, 0, False),
    ("psp_bottleneck_3x3_4096_to_512", 1, 4096, 512, 65, 129, 3, 1, 1, False),
    ("dsn_3x3_1024_to_512", 1, 1024, 512, 65, 129, 3, 1, 1, True),
]


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("shape", CONV_SHAPES, ids=[c[0] for c in CONV_SHAPES])
def test_conv_training_passes_match_float64(shape, precise):
    """Fn.Conv2d forward (TF32 or 3xTF32), data gradient and weight / bias gradients (TF32) against float64 torch."""
    import torch.nn.functional as F
    from structure_knowledge_distillation_b200 import functions as Fn, ops
    _, n, cin, cout, h, w, k, s, pad, bias = shape
    g = torch.Generator(device="cuda").manual_seed(cin + cout + k)
    x = torch.randn(n, cin, h, w, device="cuda", generator=g)
    wt = torch.randn(cout, cin, k, k, device="cuda", generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, device="cuda", generator=g) if bias else None
    xn = x.clone(memory_format=torch.channels_last).requires_grad_(True)
    wn = wt.clone(memory_format=torch.channels_last).requires_grad_(True)
    bn = b.clone().requires_grad_(True) if bias else None
    y = Fn.Conv2d.apply(xn, wn, bn, s, pad, 1, precise)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(ops.to_nhwc(dy))
    xd, wd = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    bd = b.double().requires_grad_(True) if bias else None
    yd = F.conv2d(xd, wd, bd, s, pad)
    yd.backward(dy.double())
    rep = dict(fwd=_rel(y.detach().contiguous(), yd.detach()), dgrad=_rel(xn.grad.contiguous(), xd.grad), wgrad=_rel(wn.grad.contiguous(), wd.grad))
    if bias:
        rep["bgrad"] = _rel(bn.grad, bd.grad)
    print("\nKERNEL seg", shape[0], "3xTF32" if precise else "TF32", rep)
    assert rep["fwd"] < (1e-5 if precise else 2e-3), rep
    assert rep["dgrad"] < 2e-3 and rep["wgrad"] < 2e-3 and rep.get("bgrad", 0.0) < 1e-5, rep


@pytest.mark.parametrize("c,residual", [(1024, True), (2048, True), (1024, False), (2048, False)])
def test_abn_training_at_wide_channels_matches_float64(c, residual):
    """Train-mode ABN (+ fused residual add + ReLU, or ReLU alone) at 1024 / 2048 channels: output, running statistics and every
    gradient against the float64 restatement of the reference's InPlace-ABN."""
    from oracle import port
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200.libs import InPlaceABNSync
    g = torch.Generator(device="cuda").manual_seed(c)
    n, h, w = 2, 33, 65
    x = torch.randn(n, c, h, w, device="cuda", generator=g) * 2 + 0.5
    r = torch.randn(n, c, h, w, device="cuda", generator=g) if residual else None
    bn = InPlaceABNSync(c, activation="none").cuda().train()
    ref = port.ABN(c, activation=port.ACT_NONE).cuda().double().train()
    with torch.no_grad():
        wv = 1.0 + 0.3 * torch.randn(c, device="cuda", generator=g); bv = 0.2 * torch.randn(c, device="cuda", generator=g)
        bn.weight.copy_(wv); bn.bias.copy_(bv); ref.weight.copy_(wv); ref.bias.copy_(bv)
    xn = ops.to_nhwc(x).requires_grad_(True)
    rn = ops.to_nhwc(r).requires_grad_(True) if residual else None
    y = bn(xn, residual=rn, fuse_relu=True)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(ops.to_nhwc(dy))
    xd = x.double().requires_grad_(True)
    rd = r.double().requires_grad_(True) if residual else None
    yd = torch.relu(ref(xd) + (rd if residual else 0))
    yd.backward(dy.double())
    rep = dict(fwd=_rel(y.detach().contiguous(), yd.detach()), dx=_rel(xn.grad.contiguous(), xd.grad),
               dweight=_rel(bn.weight.grad, ref.weight.grad), dbias=_rel(bn.bias.grad, ref.bias.grad),
               running_var=_rel(bn.running_var, ref.running_var))
    if residual:
        rep["dres"] = _rel(rn.grad.contiguous(), rd.grad)
    print("\nKERNEL seg abn", c, "residual" if residual else "relu", rep)
    assert max(rep.values()) < 1e-5, rep


def test_psp_pool_and_assemble_backward_at_2048_channels():
    """The PSP module's pyramid pooling and its concat assembly backward at 2048 channels against float64 adaptive pooling / bilinear
    upsampling (align_corners=True)."""
    import torch.nn.functional as F
    from structure_knowledge_distillation_b200 import functions as Fn, ops
    g = torch.Generator(device="cuda").manual_seed(7)
    n, c, h, w, cs = 2, 2048, 65, 129, 512
    sizes = (1, 2, 3, 6)
    x = torch.randn(n, c, h, w, device="cuda", generator=g)
    xn = ops.to_nhwc(x).requires_grad_(True)
    pooled = Fn.PspPool.apply(xn, sizes)
    dp = torch.randn(pooled.shape, device="cuda", generator=g)
    pooled.backward(dp)
    xd = x.double().requires_grad_(True)
    pd = torch.cat([F.adaptive_avg_pool2d(xd, s).flatten(2).transpose(1, 2) for s in sizes], 1)
    pd.backward(dp.double())
    rep = dict(pool=_rel(pooled.detach(), pd.detach()), pool_dx=_rel(xn.grad.contiguous(), xd.grad))
    stages = [torch.randn(n, s * s, cs, device="cuda", generator=g).requires_grad_(True) for s in sizes]
    feats = ops.to_nhwc(torch.randn(n, c, h, w, device="cuda", generator=g)).requires_grad_(True)
    cat = Fn.PspAssemble.apply(feats, sizes, *stages)
    dc = torch.randn(cat.shape, device="cuda", generator=g)
    cat.backward(ops.to_nhwc(dc))
    sd = [t.detach().double().requires_grad_(True) for t in stages]
    fd = feats.detach().double().requires_grad_(True)
    up = [F.interpolate(t.transpose(1, 2).reshape(n, cs, s, s), size=(h, w), mode="bilinear", align_corners=True) for t, s in zip(sd, sizes)]
    catd = torch.cat(up + [fd], 1)
    catd.backward(dc.double())
    rep["assemble"] = _rel(cat.detach().contiguous(), catd.detach())
    rep["assemble_dstages"] = max(_rel(a.grad, b.grad) for a, b in zip(stages, sd))
    rep["assemble_dfeats"] = _rel(feats.grad.contiguous(), fd.grad)
    print("\nKERNEL seg psp", rep)
    assert max(rep.values()) < 1e-5, rep


def test_forward_stages_against_float64_port():
    """Where a ResNet101 training forward departs from float64: each of the seven outputs of the first step against oracle/port.py run in
    float64 on the GPU with the same weights and dropout masks (printed; the early, fp32-grade stages are held to 1e-4)."""
    from oracle import make_golden_seg as G
    from structure_knowledge_distillation_b200 import ops
    m, src = _seg("r101_c19")
    ref = src.double().cuda().train()
    for d, mk in zip(ref.dropouts(), G.masks(src)):
        d.injected = mk.cuda()
    images, _ = G.batch(19)
    with torch.no_grad():
        want = ref(images.double().cuda())
    got = m.model.train()(ops.pad_channels(images.cuda(), 4))
    names = ("logits", "dsn", "feat", "x4", "x3", "x2", "x1")
    rep = {k: _rel(a.detach().contiguous(), b) for k, a, b in zip(names, got, want)}
    print("\nPARITY seg stages float64", rep)
    assert rep["x1"] < 1e-4 and rep["x2"] < 1e-4, rep


@pytest.mark.parametrize("name", ["r101_c19", "r101_c21", "r101_c19_ohem", "r18_c19"])
def test_step_matches_reference_golden(name):
    """Under SegModel's default policy: the loss of both steps within 1e-3 (OHEM's second step: 1e-2); the first step's logits,
    per-tensor gradient norms, sampled gradients and SGD update.  The second step is taken from parameters the first step's TF32 gradients moved, and train-mode BN at
    batch 2 amplifies that difference (DESIGN.md §4), so only its loss is held to the reference."""
    reps = _report(name)
    print("\nPARITY seg", name, "step 1", reps[0])
    print("PARITY seg", name, "step 2", reps[1])
    assert reps[0]["loss"] < TOL["loss"], reps
    assert reps[1]["loss"] < (OHEM_STEP2_LOSS if name.endswith("ohem") else TOL["loss"]), reps
    r = reps[0]
    assert r["logits"] < TOL["logits"], r
    assert r["grad_norm"][0] < TOL["grad_norm"], r
    assert r["grad_samples"] < TOL["grad_samples"], r
    assert r["update"] < TOL["update"], r


def test_precision_policies_report():
    """The three policies of DESIGN.md §4 on the 19-class ResNet101 case, printed; each keeps the first step's loss within 1e-3."""
    for policy in ("early", "layer3", "all"):
        reps = _report("r101_c19", policy)
        print("\nPARITY seg policy", policy, "step 1", reps[0])
        print("PARITY seg policy", policy, "step 2", reps[1])
        assert reps[0]["loss"] < TOL["loss"], (policy, reps)


def _dump(m):
    return [float(m.G_loss)] + [p.detach().clone() for p in m.model.parameters()] + [b.detach().clone() for b in m.model.buffers()]


def _same(a, b):
    return all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


def test_cuda_graph_replay_equals_eager_steps():
    """Three replays of the captured ResNet101 step, rewound to the starting state after the capture, equal three eager steps from that
    state bit for bit; a staged batch reaches the graph."""
    from oracle import make_golden_seg as G
    m, _ = _seg("r101_c19")
    eager = []
    for _ in range(3):
        m.optimize_parameters()
        torch.cuda.synchronize()
        eager.append(_dump(m))
    del m
    m, _ = _seg("r101_c19")
    snap = ({k: v.clone() for k, v in m.model.state_dict().items()}, m.G_solver.flat_m.clone())
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                      # eager warm-up, capture
    assert m._graphs["captured"]
    with torch.no_grad():
        cur = m.model.state_dict()
        for k, v in snap[0].items():
            cur[k].copy_(v)
        m.G_solver.flat_m.copy_(snap[1])
    for want in eager:
        m.set_input(G.batch(19))
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), want)


@pytest.mark.parametrize("kind", ["resnet101", "resnet18", "espnet_c", "espnet", "mobilenetv2"])
def test_each_network_takes_a_step(kind):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m = SegModel(make_args(batch_size=2, seg_model=kind))
    assert not any(hasattr(m, a) for a in ("teacher", "parallel_teacher", "D_model", "D_solver"))
    assert not any(isinstance(x, Discriminator) for x in m.model.modules())
    p0 = m.G_solver.flat_p.clone()
    m.set_input(port.synthetic_batch(2, 96, 128, seed=5))
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert torch.isfinite(torch.tensor(float(m.G_loss))) and float(m.G_loss) > 0
    assert not torch.equal(p0, m.G_solver.flat_p) and bool(torch.isfinite(m.G_solver.flat_p).all())


def test_launch_list_has_no_aten_compute():
    """One eager ResNet101 step under torch.profiler: every kernel is this library's, apart from copies, fills and the dropout keep-mask
    scaling (two (N, C) elementwise launches); no ATen / cuDNN / cuBLAS convolution, batch norm, softmax, upsample or GEMM."""
    from torch.profiler import ProfilerActivity, profile
    m, _ = _seg("r101_c19")
    m.optimize_parameters()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.optimize_parameters()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    foreign = [n for n in names if any(s in n for s in ("at::native", "cudnn", "cublas", "cutlass", "xmma", "sm90_xmma", "nvjet"))]
    allowed = ("copy", "Copy", "fill", "Fill", "Memcpy", "Memset")
    compute = [n for n in foreign if not any(s in n for s in allowed)]
    print("\nLAUNCHES seg resnet101: %d kernels, %d ATen/vendor, %d of them compute" % (len(names), len(foreign), len(compute)))
    for n in sorted(set(compute)):
        print("   ", compute.count(n), n[:160])
    bad = [n for n in compute if any(s in n.lower() for s in ("conv", "norm", "softmax", "upsample", "interp", "gemm", "reduce", "pool"))]
    assert not bad, bad
    # what is left: autograd's sum of two gradients where a tensor feeds two layers (a block's input: its first convolution and the
    # residual) and the dropout keep-mask scaling -- DESIGN.md §7
    assert all(("CUDAFunctor_add" in n or "MulFunctor" in n) for n in compute), sorted(set(compute))
    assert len(names) > 500


def test_checkpoint_round_trip_into_netmodel_teacher(tmp_path):
    """save_ckpt after a step -> NetModel(T_ckpt_path=...): the frozen teacher's logits equal SegModel's eval-mode logits of the same
    weights (rel-L2 1e-6)."""
    from oracle import port
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m, _ = _seg("r101_c19", snapshot_dir=str(tmp_path))
    m.optimize_parameters()
    path = m.save_ckpt(0, 1, 0.5, None)
    images, _ = port.synthetic_batch(2, 96, 128, seed=9)
    x = ops.pad_channels(images.cuda(), 4)
    with torch.no_grad():
        mine = m.model.eval()(x)[0].contiguous().clone()
    m.model.train()
    n = NetModel(make_args(batch_size=2, T_ckpt_path=path, pi=False, pa=False, ho=False))
    with torch.no_grad():
        theirs = n.teacher.eval()(x)[0].contiguous()
    err = _rel(theirs, mine)
    print("\nPARITY seg checkpoint round trip rel-L2", err)
    assert err < 1e-6


def test_full_size_step_peak_memory():
    """Batch 8 at 512x1024, ResNet101, 19 classes: one step runs and its peak allocation is reported (it must fit an 80 GB H100)."""
    from oracle import port
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = SegModel(make_args(batch_size=8, seg_model="resnet101"))
    m.set_input(port.synthetic_batch(8, 512, 1024, seed=3))
    m.optimize_parameters()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("\nMEMORY seg resnet101 b8 512x1024 peak %.2f GB, loss %.4f" % (peak / 1e9, float(m.G_loss)))
    assert torch.isfinite(torch.tensor(float(m.G_loss)))
    assert peak < 78e9


def _ddp_worker(rank, world, port_no, out):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port_no), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port
        from structure_knowledge_distillation_b200.networks.seg_model import SegModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        torch.manual_seed(100 + rank)                                  # different init per rank: SegModel broadcasts rank 0's
        m = SegModel(make_args(batch_size=1, seg_model="resnet101", sync_bn=True))
        for d in m.model.dropouts():
            d.injected = (torch.rand(1, 512, generator=torch.Generator().manual_seed(5 + rank)) >= 0.1).float()
        p0 = m.G_solver.flat_p.clone()
        m.set_input(port.synthetic_batch(1, 96, 128, seed=7 + rank))  # each rank its own shard
        m.G_solver._buckets = None                                     # one exchange after backward
        m._phase()
        local = m.G_solver.flat_g.clone()
        m.G_solver.all_reduce_grads(world)
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        ref_sum = sum(parts)
        err = float((m.G_solver.flat_g - ref_sum).norm() / ref_sum.norm())
        lr, wd = m.G_solver.param_groups[0]["lr"], m.args.weight_decay
        m.G_solver.step()
        expect = p0 - lr * (ref_sum / world + wd * p0)
        err2 = float((m.G_solver.flat_p - expect).norm() / (lr * (ref_sum / world + wd * p0)).norm())
        pg = m.G_solver.flat_p.clone()
        allp = [torch.empty_like(pg) for _ in range(world)]
        dist.all_gather(allp, pg)
        same = all(torch.equal(t, allp[0]) for t in allp)
        if rank == 0:
            out.put(("ok" if err < 1e-6 and err2 < 1e-5 and same else "fail", err, err2, same))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step():
    """ResNet101 with sync_bn over 2 NCCL ranks: the all-reduced gradient is the sum of the shards', the step applies their mean and the
    replicas stay identical.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_ddp_worker, args=(2, 29641, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY seg_dp_world2", res)
    assert res[0] == "ok", res
