"""Channel-wise distillation (CWD) on the H100: the csrc/cwd.cu kernels against float64 autograd over layouts, widths and grids, exact
zeros, repeatability, NetModel steps against tests/golden/cwd.pt.gz (oracle/cwd_port.py), CUDA-graph replay, the training-state file
and resume, the defaults launching none of it, and two NCCL ranks."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _relf(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _map(n, c, h, w, gen, layout, pitch=None, scale=1.0):
    """(N, C, H, W) random map: "nchw" contiguous, or "nhwc" rows -- the last c channels of `pitch`-wide rows when given (the teacher's
    x4 is such a slice of the PSP concat buffer; an odd pitch leaves the slice misaligned and takes the scalar path)."""
    if layout == "nchw":
        return torch.randn(n, c, h, w, generator=gen, device="cuda") * scale
    p = pitch or c
    buf = torch.randn(n, h, w, p, generator=gen, device="cuda") * scale
    return buf.permute(0, 3, 1, 2)[:, p - c:]


def _ref(S, T, tau):
    from oracle import cwd_port as P
    sd = S.detach().double().requires_grad_(True)
    loss = P.cwd_loss(sd, T.double(), tau)
    (g,) = torch.autograd.grad(loss, sd)
    return loss, g


def _run(S, T, tau, gscale=1.0):
    from structure_knowledge_distillation_b200 import functions as Fn
    Sg = S.detach().requires_grad_(True)
    loss = Fn.ChannelWiseLoss.apply(Sg, T, tau)
    (g,) = torch.autograd.grad(loss * gscale, Sg)
    return loss, g


# (N, C, H, W, layout, student pitch, teacher pitch, scale, tau)
CASES = [
    (2, 11, 33, 65, "nchw", None, None, 1.0, 4.0),
    (2, 19, 65, 129, "nhwc", 20, 20, 3.0, 4.0),          # the logits as the networks carry them: 19 of 20 channels, scalar path
    (2, 19, 65, 129, "nchw", None, None, 3.0, 4.0),
    (1, 21, 17, 23, "nhwc", None, None, 1.0, 1.0),
    (2, 150, 33, 41, "nhwc", None, None, 2.0, 4.0),
    (2, 150, 13, 17, "nchw", None, None, 2.0, 2.0),      # prime H and W
    (2, 64, 33, 65, "nhwc", None, None, 1.0, 4.0),
    (2, 512, 17, 31, "nhwc", None, None, 1.0, 4.0),
    (1, 2048, 17, 31, "nhwc", None, 4096, 1.0, 4.0),     # teacher x4: a channel slice of the PSP concat buffer
    (2, 64, 9, 13, "nhwc", None, 67, 1.0, 4.0),          # teacher 3 floats into a 67-wide buffer: misaligned, scalar path
    (3, 19, 1, 1, "nhwc", 20, None, 1.0, 4.0),           # HW = 1
    (1, 256, 129, 257, "nhwc", None, None, 1.0, 4.0),    # x1 at 512x1024
    (1, 19, 360, 480, "nhwc", 20, 20, 3.0, 4.0),         # the full ESPNet's input-resolution logits
    (1, 19, 360, 480, "nchw", None, None, 3.0, 4.0),
    (2, 19, 65, 129, "nhwc", 20, 20, 300.0, 4.0),        # logits x100: most pS underflow to 0 in fp32, log pS stays finite
    (2, 19, 33, 65, "nchw", None, None, 300.0, 1.0),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N%d_C%d_%dx%d_%s_p%s-%s_x%g_t%g" % c)
def test_kernels_match_float64(case):
    """Loss and student gradient against autograd through F.log_softmax in float64.  Bound: z = x / tau and z - lse run in double and
    the sums of exponentials and of the KL terms accumulate in double, so the only fp32 roundings are those of the exponent argument
    (relative 2^-24, i.e. |z - lse| * 6e-8 absolute) and of expf (2 ulp): each pT or pS is within (2 + |z - lse|) * 6e-8 relative.
    Only positions with |z - lse| below ~100 carry weight (e^-100 is nothing), so each term is within ~1e-5 relative, and the loss, a
    sum of non-negative per-channel KLs, and dS = tau / (N*C) (pS - pT) within that relative to their size: 1e-4 is held with margin.
    Independent S and T keep the loss free of cancellation."""
    n, c, h, w, layout, ps, pt, scale, tau = case
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + c * 7 + h + w)
    S = _map(n, c, h, w, gen, layout, ps, scale)
    T = _map(n, c, h, w, gen, layout, pt, scale)
    loss, g = _run(S, T, tau, 3.0)
    ref, gref = _ref(S, T, tau)
    assert torch.isfinite(loss) and bool(torch.isfinite(g).all())
    if h * w == 1:
        assert float(loss) == 0.0 and torch.count_nonzero(g) == 0
        return
    e_loss, e_grad = _relf(loss, ref), _rel(g.double(), 3.0 * gref)
    print("\nPARITY cwd", case, "loss %.3e (%.6g) grad %.2e" % (e_loss, float(ref), e_grad))
    assert e_loss < 1e-4 and e_grad < 1e-4, (e_loss, e_grad)
    assert g.stride() == S.stride()                               # the gradient keeps the student's layout


@pytest.mark.parametrize("layout, c, pitch", [("nhwc", 64, None), ("nhwc", 19, 20), ("nchw", 19, None), ("nhwc", 1, None)])
def test_equal_maps_give_exact_zeros(layout, c, pitch):
    """S = T bit for bit: both softmaxes are the same numbers, so every KL term and every pS - pT is exactly 0 (float4, scalar and
    pixel-lane mappings)."""
    gen = torch.Generator(device="cuda").manual_seed(11)
    S = _map(2, c, 17, 23, gen, layout, pitch, 5.0)
    T = S.detach().clone()
    for tau in (4.0, 3.0):
        loss, g = _run(S, T, tau)
        assert float(loss) == 0.0 and torch.count_nonzero(g) == 0, (tau, float(loss))


def test_single_position_gives_exact_zeros():
    """HW = 1: each softmax is 1 whatever the values, so the loss and the gradient are exactly 0, at any temperature."""
    gen = torch.Generator(device="cuda").manual_seed(12)
    for layout, c in (("nhwc", 512), ("nchw", 19), ("nhwc", 7)):
        S, T = _map(4, c, 1, 1, gen, layout, None, 10.0), _map(4, c, 1, 1, gen, layout, None, 10.0)
        for tau in (4.0, 3.0, 0.7):
            loss, g = _run(S, T, tau)
            assert float(loss) == 0.0 and torch.count_nonzero(g) == 0, (layout, c, tau, float(loss))


def test_repeatable_and_alignment_independent():
    """Two calls give bit-identical loss and dS.  The same values read through the float4 path (aligned rows) and through the scalar
    path (the same rows one float into a wider buffer) give the same bits too: each channel is summed in the same order on both."""
    gen = torch.Generator(device="cuda").manual_seed(13)
    n, c, h, w = 2, 256, 65, 129
    S, T = _map(n, c, h, w, gen, "nhwc"), _map(n, c, h, w, gen, "nhwc")
    runs = [_run(S, T, 4.0) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    bufS = torch.zeros(n, h, w, c + 1, device="cuda"); bufT = torch.zeros(n, h, w, c + 1, device="cuda")
    bufS[..., 1:] = S.permute(0, 2, 3, 1); bufT[..., 1:] = T.permute(0, 2, 3, 1)
    S1, T1 = bufS.permute(0, 3, 1, 2)[:, 1:], bufT.permute(0, 3, 1, 2)[:, 1:]
    loss1, g1 = _run(S1, T1, 4.0)
    assert torch.equal(loss1, runs[0][0]) and torch.equal(g1, runs[0][1])


# -------------------------------------------------------------------------------------------- NetModel steps against the golden
def _case_model(spec):
    from oracle import make_golden_cwd as G, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**spec["cfg"])
    teacher, student, D, mimic, cwd, images, labels, masks, alpha = G.case_inputs(spec)
    kw = dict(cwd=True, lambda_cwd=spec["lambda_cwd"], lambda_cwd_feat=spec["cwd_feat"])
    if spec["mimic"] is not None:
        kw.update(mimic=True, lambda_mimic=spec["mimic"])
    m = NetModel(make_args(batch_size=spec["batch"], pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, student=spec["kind"], **kw))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for mine, ref in ((m.mimic_adapters, mimic), (m.cwd_adapters, cwd)):
        if mine is not None:
            mine.load_state_dict(ref.state_dict())
        else:
            assert len(ref) == 0
    for drop, mk in zip(m.student.dropouts(), masks):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = alpha.cuda()
    m.set_input((images, labels, None, None))
    return m, c


def _samples(named, digest):
    """(mine, gold) rows of sampled values normalised by the golden's norm, and the worst relative norm error."""
    worst, mine_s, gold_s = 0.0, [], []
    for name, v in named:
        gd = digest.get(name)
        if gd is None or gd["norm"] < 1e-6:
            continue
        a = v.detach().flatten().double()
        worst = max(worst, abs(float(a.norm()) - gd["norm"]) / gd["norm"])
        mine_s.append(a[gd["idx"].to(a.device)].cpu() / gd["norm"]); gold_s.append(gd["samples"].double() / gd["norm"])
    return torch.cat(mine_s), torch.cat(gold_s), worst


@pytest.mark.parametrize("name", ["r18_pi_pa_ho_cwd_logits_512_b1", "r18_cwd_levels_mimic_x3_96x128_b2", "espnet_cwd_logits_360x480_b1",
                                  "espnet_c_cwd_psp_360x480_b1"])
def test_step_matches_golden(name):
    """Losses, logits, sampled student and adapter gradients (both families) and the parameters after one SGD step against the fp32 CPU
    restatement.  Bounds are tests/test_feature_kd_gpu.py's: the random-init student runs TF32 convolutions whose rounding batch-statistic
    BN amplifies, so gradients agree in direction and norm, not to fp32.  The task and Pi losses agree to 1e-3, MIMIC to 5e-3 and the
    CWD terms -- KLs of softmaxes of those logits and adapted features -- to 1e-2; the adapters' gradients, one 1x1 layer from the
    loss, to 0.1."""
    from oracle import make_golden_cwd as G
    gold = G.load()[name]
    m, cfg = _case_model(G.GOLDEN_CASES[name])
    fams = [(f, a) for f, a in (("mimic", m.mimic_adapters), ("cwd", m.cwd_adapters)) if a is not None]
    p0 = {(f, k): p.detach().clone() for f, a in [("student", m.student)] + fams for k, p in a.named_parameters()}
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    rep = dict(ce=_relf(m.mc_G_loss, gold["ce"]), G=_relf(m.G_loss, gold["G"]))
    if cfg.pi:
        rep["pi"] = _relf(m.pi_G_loss, gold["pi"])
    if cfg.pa:
        rep["pa"] = _relf(m.pa_G_loss, gold["pa"])
    for term in ("mimic", "cwd"):
        if term not in gold:
            continue
        mine, ref = getattr(m, term + "_G_loss"), gold[term]
        mine, ref = (mine, ref) if isinstance(ref, list) else ([mine], [ref])
        assert len(mine) == len(ref)
        for ind, (a, b) in enumerate(zip(mine, ref)):
            if b == 0.0:
                assert a == 0.0 and isinstance(a, float)
            else:
                rep["%s%d" % (term, ind)] = _relf(a, b)
    rep["logits_S"] = _rel(m.preds_S[0][:, :, ::8, ::8].float().cpu(), gold["logits_S"])
    parts = [("student", m.student, gold["student_grads"], gold["student_update"])] + \
        [(f, a, gold[f + "_adapter_grads"], gold[f + "_adapter_update"]) for f, a in fams]
    for what, mod, digest, _ in parts:
        sm, sg, worst = _samples([(k, p.grad) for k, p in mod.named_parameters()], digest)
        rep[what + "_grad_norm"], rep[what + "_grad_l2"] = worst, float((sm - sg).norm() / sg.norm())
        rep[what + "_grad_cos"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    m.G_solver.step()
    for what, mod, digest, update in parts:
        mine, ref = [], []
        for k, p in mod.named_parameters():
            if k in update and digest[k]["norm"] >= 1e-6:
                d = (p.detach() - p0[(what, k)]).flatten().double()[digest[k]["idx"].to(p.device)].cpu()
                mine.append(d / digest[k]["norm"]); ref.append(update[k].double() / digest[k]["norm"])
        a, b = torch.cat(mine), torch.cat(ref)
        rep[what + "_update_l2"] = float((a - b).norm() / b.norm())
    print("\nPARITY cwd step", name, {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        if k in ("ce", "pi", "G"):
            assert v < 1e-3, (k, v)
        elif k == "pa" or k.startswith("mimic") and not k.startswith("mimic_"):
            assert v < 5e-3, (k, v)
        elif k.startswith("cwd") and not k.startswith("cwd_"):
            assert v < 1e-2, (k, v)
    assert rep["logits_S"] < 3e-2
    assert rep["student_grad_norm"] < 0.6 and rep["student_grad_l2"] < 0.35 and rep["student_grad_cos"] > 0.93
    assert rep["student_update_l2"] < 0.35
    for f, _ in fams:
        assert rep[f + "_grad_norm"] < 0.1 and rep[f + "_grad_l2"] < 0.1 and rep[f + "_grad_cos"] > 0.99, f
        assert rep[f + "_update_l2"] < 0.1, f


# -------------------------------------------------------------------------------------------- graphs, repeatability, state, ranks
def _resnet18(batch, h, w, cfg, without=(), **extra):
    """NetModel with the ResNet18 student on the seeded weights, dropout masks, WGAN-GP alpha and batch of the golden cases; the
    argument fields named in `without` are removed, as in a namespace written before they existed."""
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**cfg)
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    torch.manual_seed(21)                                                  # the adapters' init
    args = make_args(batch_size=batch, pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, **extra)
    for f in without:
        delattr(args, f)
    m = NetModel(args)
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for drop, mk in zip(m.student.dropouts(), cases.dropout_masks(student, batch, seed=2)):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    return m


GRAPH_CFG = dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")
GRAPH_EXTRA = dict(cwd=True, lambda_cwd=3.0, lambda_cwd_feat=[0.0, 0.0, 0.0, 1.0, 1.0], mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0],
                   overlap_streams=False)


def _terms(v):
    return [float(t) for t in v] if isinstance(v, list) else [float(v)]


def _adapters(m):
    return [a for a in (m.mimic_adapters, m.cwd_adapters) if a is not None]


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + _terms(m.cwd_G_loss) + [p.detach().clone() for p in m.student.parameters()] + \
        [p.detach().clone() for a in _adapters(m) for p in a.parameters()] + [b.detach().clone() for b in m.student.buffers()]


def _same(a, b):
    return len(a) == len(b) and all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


def _mods(m):
    return [m.student, m.D_model] + _adapters(m)


def _state(m):
    return [{k: v.clone() for k, v in mod.state_dict().items()} for mod in _mods(m)] + [m.G_solver.flat_m.clone(), m.D_solver.flat_m.clone()]


def _rewind(m, snap):
    mods = _mods(m)
    with torch.no_grad():
        for mod, sd in zip(mods, snap[:len(mods)]):
            cur = mod.state_dict()
            for k, v in sd.items():
                cur[k].copy_(v)                                           # in place: the captured graph reads these buffers
        m.G_solver.flat_m.copy_(snap[-2]); m.D_solver.flat_m.copy_(snap[-1])


def test_cuda_graph_replays_equal_eager_and_runs_repeat():
    """ResNet18 Pi + Pa + Ho + CWD on the logits, x4 (512 -> 2048) and the PSP features, MIMIC at x4 as well, 256x256 batch 2,
    overlap_streams off: two eager runs of three steps are bitwise equal, and three replays of the captured step, rewound to the
    starting state, equal them."""
    runs = []
    for _ in range(2):
        m = _resnet18(2, 256, 256, GRAPH_CFG, **GRAPH_EXTRA)
        want = []
        for _ in range(3):
            m.optimize_parameters()
            torch.cuda.synchronize()
            want.append(_dump(m))
        runs.append(want)
        del m
    assert all(_same(a, b) for a, b in zip(*runs))
    m = _resnet18(2, 256, 256, GRAPH_CFG, **GRAPH_EXTRA)
    snap = _state(m)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()
    assert m._graphs["captured"]
    _rewind(m, snap)
    for w in runs[0]:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)


BASE_KEYS = {"format", "version", "world_size", "kind", "classes_num", "step", "epoch", "best_mean_IU", "IU_array", "ranks",
             "state_dict", "D_state_dict", "G_solver", "D_solver"}


def test_training_state_keys_and_resume(tmp_path):
    """A model with CWD feature levels writes `cwd_state_dict` beside `mimic_state_dict`; CWD on the logits alone adds no key.  Three
    steps, a save, a load into a fresh CUDA-graph model and three more steps equal six uninterrupted steps bit for bit.  A MIMIC-only
    file (the layout written before CWD existed) loads into a MIMIC-only model, and a CWD file is refused by a model without CWD."""
    cfg = dict(pi=True, pa=True, ho=True, adv_type="hinge")
    extra = dict(cwd=True, lambda_cwd_feat=[0.0, 0.0, 0.0, 1.0, 1.0], mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0], overlap_streams=False)
    logits_only = _resnet18(1, 256, 256, cfg, cwd=True)
    assert logits_only.cwd_adapters is None
    logits_only.save_training_state(str(tmp_path / "logits.pth"), 0)
    assert set(torch.load(str(tmp_path / "logits.pth"), weights_only=False)) == BASE_KEYS
    del logits_only
    mimic_only = _resnet18(1, 256, 256, cfg, mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0])
    mimic_only.optimize_parameters()
    mimic_only.save_training_state(str(tmp_path / "mimic.pth"), 1)
    assert set(torch.load(str(tmp_path / "mimic.pth"), weights_only=False)) == BASE_KEYS | {"mimic_state_dict"}
    del mimic_only
    again = _resnet18(1, 256, 256, cfg, mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0])
    assert again.load_training_state(str(tmp_path / "mimic.pth")) == 1
    del again
    want = []
    m = _resnet18(1, 256, 256, cfg, **extra)
    for k in range(6):
        m.optimize_parameters()
        if k == 2:
            m.save_training_state(str(tmp_path / "cwd.pth"), 3)
        if k >= 3:
            torch.cuda.synchronize()
            want.append(_dump(m))
    ck = torch.load(str(tmp_path / "cwd.pth"), weights_only=False)
    assert set(ck) == BASE_KEYS | {"mimic_state_dict", "cwd_state_dict"}
    assert set(ck["cwd_state_dict"]) == {"level3.weight", "level3.bias", "level4.weight", "level4.bias"}
    assert set(ck["mimic_state_dict"]) == {"level3.weight", "level3.bias"}
    del m
    m = _resnet18(1, 256, 256, cfg, **extra)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                   # captured
    assert m._graphs["captured"]
    assert m.load_training_state(str(tmp_path / "cwd.pth")) == 3
    for w in want:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)
    other = _resnet18(1, 256, 256, cfg, mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0])
    with pytest.raises(ValueError, match="G_solver.numel|cwd_state_dict"):
        other.load_training_state(str(tmp_path / "cwd.pth"))


def test_defaults_launch_no_cwd_kernel(monkeypatch):
    """With make_args' defaults (cwd off, whatever lambda_cwd_feat holds) no CWD kernel runs and no CWD adapter exists; G_solver's
    flat buffer and the state keys are those of a run without the CWD fields, with and without MIMIC adapters."""
    from structure_knowledge_distillation_b200 import ops

    def refuse(*a, **k):
        raise AssertionError("a CWD kernel ran with the term off")
    for fn in ("cwd_fwd", "cwd_bwd"):
        monkeypatch.setattr(ops, fn, refuse)
    cfg = dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    fields = ("cwd", "lambda_cwd", "lambda_cwd_feat", "cwd_tau")
    for extra in ({}, dict(mimic=True, lambda_mimic=[0.0, 0.0, 1.0, 1.0])):
        old = _resnet18(1, 256, 256, cfg, without=fields, **extra)
        layout = (old.G_solver.flat_p.numel(), [tuple(p.shape) for p in old.G_solver.params], set(old._extra_states()))
        del old
        for more in ({}, dict(lambda_cwd_feat=[1.0] * 5)):
            m = _resnet18(1, 256, 256, cfg, **extra, **more)
            m.optimize_parameters()
            torch.cuda.synchronize()
            assert m.cwd_adapters is None and m.cwd_G_loss is None
            trained = [p for p in m.student.parameters() if p.requires_grad] + \
                ([p for p in m.mimic_adapters.parameters()] if m.mimic_adapters is not None else [])
            assert len(m.G_solver.params) == len(trained) and all(a is b for a, b in zip(m.G_solver.params, trained))
            assert (m.G_solver.flat_p.numel(), [tuple(p.shape) for p in m.G_solver.params], set(m._extra_states())) == layout
            del m


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
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, cwd=True,
                               lambda_cwd_feat=[0.0, 0.0, 0.0, 1.0]))
        for d in m.student.dropouts():
            d.injected = (torch.rand(1, 128, generator=torch.Generator().manual_seed(5 + rank)) >= 0.1).float()
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
        lo = m.G_solver._offsets[sum(1 for p in m.student.parameters() if p.requires_grad)]   # the adapters follow the student
        ad_err = float((summed[lo:] - ref_sum[lo:]).norm() / ref_sum[lo:].norm())
        if rank == 0:
            out.put(("ok", err, ad_err, [float(v) for v in m.cwd_G_loss]))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_sums_the_shard_gradients():
    """ResNet18 with CWD on the logits and at x4 over 2 NCCL ranks: the all-reduced flat gradient (the CWD adapter included) is the sum
    of the per-rank gradients.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29653, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY cwd world2", res)
    assert res[0] == "ok" and res[2] < 1e-6, res
