"""Intra-class feature variation distillation (IFV) on the H100: the csrc/ifv.cu kernels against float64 autograd of oracle/ifv_port.py
over class counts, widths, layouts and grids, the nearest label map bit for bit, exact zeros, repeatability, NetModel steps against
tests/golden/ifv.pt.gz, CUDA-graph replay, the training-state file and resume, the defaults launching none of it, and two NCCL ranks."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _relf(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _map(n, c, h, w, gen, pitch=None, off=0, scale=1.0):
    """(N, C, H, W) view of NHWC rows: channels off .. off + c of `pitch`-wide rows (dense when pitch is None).  The teacher's x4 is such
    a slice of the PSP concat buffer, ESPNet's b1 / b2 / b3 slices of theirs; an odd pitch or offset leaves it misaligned (scalar
    loads)."""
    p = pitch or c
    buf = torch.randn(n, h, w, p, generator=gen, device="cuda") * scale
    return buf.permute(0, 3, 1, 2)[:, off:off + c]


def _labels(n, H, W, K, seed, ignore=0.05, classes=None):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, classes or K, (n, H, W), generator=g)
    lab[torch.rand(n, H, W, generator=g) < ignore] = 255
    return lab.cuda()


def _ref(S, T, labels, K):
    from oracle import ifv_port as P
    sd = S.detach().double().requires_grad_(True)
    loss = P.ifv_loss(sd, T.double(), labels, K)
    (g,) = torch.autograd.grad(loss, sd)
    return loss, g


def _run(S, T, labels, K, gscale=1.0):
    from structure_knowledge_distillation_b200 import functions as Fn
    Sg = S.detach().requires_grad_(True)
    loss = Fn.IntraClassVariationLoss.apply(Sg, T, labels, K)
    (g,) = torch.autograd.grad(loss * gscale, Sg)
    return loss, g


@pytest.mark.parametrize("H, W, h, w", [(512, 512, 65, 65), (512, 1024, 65, 129), (512, 1024, 129, 257), (769, 769, 97, 97),
                                        (360, 480, 45, 60), (360, 480, 46, 61), (96, 128, 12, 16), (96, 128, 24, 32), (17, 23, 17, 23),
                                        (20, 30, 40, 60), (33, 41, 7, 5)])
def test_labels_nearest_is_f_interpolate(H, W, h, w):
    """ops.labels_nearest picks exactly the labels F.interpolate(mode="nearest") picks (the same fp32 product, floor and clamp)."""
    from structure_knowledge_distillation_b200 import ops
    lab = _labels(2, H, W, 255, H * W, ignore=0.1)
    got = ops.labels_nearest(lab, h, w)
    want = F.interpolate(lab[:, None].float(), (h, w), mode="nearest")[:, 0].long()
    assert got.dtype == torch.int32 and torch.equal(got.long(), want)


def test_labels_nearest_random_sweep():
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator().manual_seed(5)
    for _ in range(40):
        H, W = (int(v) for v in torch.randint(1, 1100, (2,), generator=g))
        h, w = (int(v) for v in torch.randint(1, 300, (2,), generator=g))
        lab = torch.randint(0, 256, (1, H, W), generator=g).cuda()
        want = F.interpolate(lab[:, None].float(), (h, w), mode="nearest")[:, 0].long()
        assert torch.equal(ops.labels_nearest(lab, h, w).long(), want), (H, W, h, w)


# (N, K, C_S, C_T, h, w, H, W, S (pitch, offset), T (pitch, offset), label classes drawn (None: all K))
CASES = [
    (2, 19, 128, 512, 65, 129, 512, 1024, (None, 0), (None, 0), None),        # the PSP level at 512x1024, float4 path
    (2, 2, 64, 64, 33, 41, 264, 328, (None, 0), (None, 0), None),
    (2, 11, 96, 160, 31, 37, 248, 296, (None, 0), (200, 40), None),           # prime grid, T an aligned slice
    (1, 21, 128, 512, 41, 41, 321, 321, (131, 3), (None, 0), None),           # VOC's count, S misaligned: scalar path
    (2, 150, 128, 256, 33, 41, 264, 328, (None, 0), (None, 0), None),         # ADE20K's count: 13 class groups, absent classes
    (1, 19, 64, 256, 129, 257, 512, 1024, (None, 0), (None, 0), None),        # x1 at 512x1024: ResNet18's 64 against the teacher's 256
    (1, 19, 512, 2048, 17, 31, 136, 248, (None, 0), (4096, 2048), None),      # teacher x4 inside the PSP concat buffer
    (2, 19, 19, 35, 23, 29, 184, 232, (None, 0), (None, 0), None),            # widths not a multiple of 4
    (2, 19, 64, 128, 13, 17, 104, 136, (131, 64), (259, 131), None),          # ESPNet-like slices: S aligned, T misaligned
    (2, 19, 128, 512, 45, 60, 360, 480, (None, 0), (None, 0), 7),             # classes 7..18 absent
    (3, 255, 32, 48, 19, 23, 152, 184, (None, 0), (None, 0), None),           # the largest class count
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N%d_K%d_S%d_T%d_%dx%d_from%dx%d_S%s-%s_T%s-%s_cls%s" % (
    c[:8] + c[8] + c[9] + (c[10],)))
def test_kernels_match_float64(case):
    """Loss and student gradient against float64 autograd of the port.  Bound: the class sums, dot products and norms accumulate in
    double, so the only roundings that matter are fp32 ones: the prototypes (kept as fp32, 2^-24 relative per component), the kept
    cos_S, cos_S - cos_T and |f_S| (2^-24 each) and dS itself.  Each cosine is within ~3 * 6e-8 absolute, so d = cos_S - cos_T (of
    order 0.1 .. 1 for independent maps) and the loss, a mean of d^2, are within ~1e-6 relative; each of the three terms of dS is within
    ~4 * 6e-8 relative and they cancel by at most a factor ~10, so dS is within ~3e-6 relative in norm.  1e-5 is held with margin."""
    n, K, cs, ct, h, w, H, W, (sp, so), (tp, to), classes = case
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + K * 7 + h + w)
    S = _map(n, cs, h, w, gen, sp, so)
    T = _map(n, ct, h, w, gen, tp, to)
    labels = _labels(n, H, W, K, K + h, classes=classes)
    loss, g = _run(S, T, labels, K, 3.0)
    ref, gref = _ref(S, T, labels, K)
    assert torch.isfinite(loss) and bool(torch.isfinite(g).all())
    e_loss, e_grad = _relf(loss, ref), _rel(g.double(), 3.0 * gref)
    print("\nPARITY ifv", case, "loss %.3e (%.6g) grad %.2e" % (e_loss, float(ref), e_grad))
    assert e_loss < 1e-5 and e_grad < 1e-5, (e_loss, e_grad)
    lab = F.interpolate(labels[:, None].float(), (h, w), mode="nearest")[:, 0]
    ignored = (lab == 255)[:, None].expand_as(g)
    assert torch.count_nonzero(g[ignored]) == 0                    # ignored pixels: exactly 0


def test_zero_feature_vector_follows_torch():
    """An all-zero student pixel: torch's cosine_similarity gives cos = 0 there and the gradient p_hat / eps (eps = 1e-8, so ~1e8 times
    the upstream gradient); the kernels do the same.  The pixel and the rest of the map are compared separately, each to 1e-5."""
    gen = torch.Generator(device="cuda").manual_seed(31)
    S = _map(2, 64, 17, 23, gen)
    T = _map(2, 128, 17, 23, gen)
    S[1, :, 5, 7] = 0.0
    labels = _labels(2, 136, 184, 19, 32)
    labels[1, 40:48, 56:64] = 3                                      # the zero pixel's label, not ignored
    loss, g = _run(S, T, labels, 19)
    ref, gref = _ref(S, T, labels, 19)
    assert _relf(loss, ref) < 1e-5
    pix = g[1, :, 5, 7].double()
    mask = torch.ones_like(g, dtype=torch.bool)
    mask[1, :, 5, 7] = False
    assert float(gref[1, :, 5, 7].norm()) > 1e4 * float(gref[mask].abs().max())             # p_hat / eps dominates
    assert _rel(pix, gref[1, :, 5, 7]) < 1e-5 and _rel(g[mask].double(), gref[mask]) < 1e-5


@pytest.mark.parametrize("cs, pitch, off", [(128, None, 0), (19, None, 0), (64, 131, 3)])
def test_equal_maps_give_exact_zeros(cs, pitch, off):
    """S = T bit for bit (also through another layout of the same values): both prototypes and both cosines are the same numbers, so
    every d, the loss, both backward class sums and dS are exactly 0."""
    gen = torch.Generator(device="cuda").manual_seed(11)
    S = _map(2, cs, 17, 23, gen, pitch, off, 5.0)
    labels = _labels(2, 136, 184, 19, 12)
    for T in (S.detach().clone(), S.detach().contiguous(memory_format=torch.channels_last)):
        loss, g = _run(S, T, labels, 19)
        assert float(loss) == 0.0 and torch.count_nonzero(g) == 0, float(loss)


def test_all_ignored_labels_give_exact_zeros():
    gen = torch.Generator(device="cuda").manual_seed(13)
    S, T = _map(2, 128, 17, 23, gen), _map(2, 512, 17, 23, gen)
    labels = torch.full((2, 136, 184), 255, dtype=torch.long, device="cuda")
    for K in (19, 150):
        loss, g = _run(S, T, labels, K)
        assert float(loss) == 0.0 and torch.count_nonzero(g) == 0


def test_repeatable_and_alignment_independent():
    """Two calls give bit-identical loss and dS.  The same values read through the float4 path (aligned rows) and through the scalar
    path (the same rows one float into wider buffers) give the same bits too: every lane owns the same channels on both paths."""
    gen = torch.Generator(device="cuda").manual_seed(14)
    n, cs, ct, h, w = 2, 128, 512, 65, 129
    S, T = _map(n, cs, h, w, gen), _map(n, ct, h, w, gen)
    labels = _labels(n, 512, 1024, 19, 15)
    runs = [_run(S, T, labels, 19) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    bufS = torch.zeros(n, h, w, cs + 1, device="cuda"); bufT = torch.zeros(n, h, w, ct + 1, device="cuda")
    bufS[..., 1:] = S.permute(0, 2, 3, 1); bufT[..., 1:] = T.permute(0, 2, 3, 1)
    S1, T1 = bufS.permute(0, 3, 1, 2)[:, 1:], bufT.permute(0, 3, 1, 2)[:, 1:]
    loss1, g1 = _run(S1, T1, labels, 19)
    assert torch.equal(loss1, runs[0][0]) and torch.equal(g1, runs[0][1])


def test_ops_refuse_bad_inputs():
    from structure_knowledge_distillation_b200 import ops
    S, T = torch.zeros(2, 8, 5, 6, device="cuda"), torch.zeros(2, 16, 5, 6, device="cuda")
    lab = torch.zeros(2, 40, 48, dtype=torch.long, device="cuda")
    with pytest.raises(ValueError, match="differ in batch or grid"):
        ops.ifv_fwd(S, torch.zeros(2, 16, 5, 7, device="cuda"), lab, 19)
    with pytest.raises(ValueError, match="labels"):
        ops.ifv_fwd(S, T, lab.int(), 19)
    with pytest.raises(ValueError, match="labels hold"):
        ops.ifv_fwd(S, T, lab[:1], 19)
    for k in (0, 256):
        with pytest.raises(ValueError, match="class count"):
            ops.ifv_fwd(S, T, lab, k)


# -------------------------------------------------------------------------------------------- NetModel steps against the golden
def _case_model(spec):
    from oracle import make_golden_ifv as G, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**spec["cfg"])
    teacher, student, D, images, labels, masks, alpha = G.case_inputs(spec)
    kw = dict(ifv=True, lambda_ifv=spec["ifv"], classes_num=spec["classes"])
    if spec["lambda_cwd"] != 0.0:
        kw.update(cwd=True, lambda_cwd=spec["lambda_cwd"])
    m = NetModel(make_args(batch_size=spec["batch"], pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, student=spec["kind"], **kw))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for drop, mk in zip(m.student.dropouts() if masks else [], masks):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = alpha.cuda()
    m.set_input((images, labels, None, None))
    return m, c


def _samples(named, digest):
    """(mine, gold) rows of sampled values normalised by the golden's norm, and the worst relative norm error.  Gradients below 1e-3 of
    the median norm are left out, as tests/test_mobilenet_gpu.py leaves them out: biases that reach the loss only through linear layers
    and a train-mode BatchNorm vanish analytically, their stored norms are cancellation residue (MobileNetV2's projection shifts)."""
    import statistics
    floor = max(1e-6, 1e-3 * statistics.median(v["norm"] for v in digest.values()))
    worst, mine_s, gold_s = 0.0, [], []
    for name, v in named:
        gd = digest.get(name)
        if gd is None or gd["norm"] < floor:
            continue
        a = v.detach().flatten().double()
        worst = max(worst, abs(float(a.norm()) - gd["norm"]) / gd["norm"])
        mine_s.append(a[gd["idx"].to(a.device)].cpu() / gd["norm"]); gold_s.append(gd["samples"].double() / gd["norm"])
    return torch.cat(mine_s), torch.cat(gold_s), worst


@pytest.mark.parametrize("name", ["r18_pi_pa_ho_ifv_psp_512_b1", "r18_ifv_levels_cwd_96x128_b2", "espnet_c_ifv_psp_360x480_b1",
                                  "mbv2_ifv_psp_voc21_96x128_b2"])
def test_step_matches_golden(name):
    """Losses, logits, sampled student gradients and the parameters after one SGD step against the fp32 CPU restatement.  Bounds are
    tests/test_cwd_gpu.py's: the random-init student runs TF32 convolutions whose rounding batch-statistic BN amplifies, so gradients
    agree in direction and norm, not to fp32.  The task and Pi losses agree to 1e-3, CWD to 1e-2, and the IFV terms -- squared
    differences of cosines of those features to their class means -- to 2e-2."""
    import statistics
    from oracle import make_golden_ifv as G
    gold = G.load()[name]
    m, cfg = _case_model(G.GOLDEN_CASES[name])
    p0 = {k: p.detach().clone() for k, p in m.student.named_parameters()}
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    rep = dict(ce=_relf(m.mc_G_loss, gold["ce"]), G=_relf(m.G_loss, gold["G"]))
    if cfg.pi:
        rep["pi"] = _relf(m.pi_G_loss, gold["pi"])
    if cfg.pa:
        rep["pa"] = _relf(m.pa_G_loss, gold["pa"])
    for term in ("cwd", "ifv"):
        if term not in gold:
            continue
        mine, ref = getattr(m, term + "_G_loss"), gold[term]
        mine, ref = (mine, ref) if isinstance(ref, list) else ([mine], [ref])
        assert len(mine) == len(ref)
        for ind, (a, b) in enumerate(zip(mine, ref)):
            rep["%s%d" % (term, ind)] = _relf(a, b)
    rep["logits_S"] = _rel(m.preds_S[0][:, :, ::8, ::8].float().cpu(), gold["logits_S"])
    sm, sg, worst = _samples([(k, p.grad) for k, p in m.student.named_parameters()], gold["student_grads"])
    rep["grad_norm"], rep["grad_l2"] = worst, float((sm - sg).norm() / sg.norm())
    rep["grad_cos"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    m.G_solver.step()
    mine, ref = [], []
    digest, update = gold["student_grads"], gold["student_update"]
    floor = max(1e-6, 1e-3 * statistics.median(v["norm"] for v in digest.values()))
    for k, p in m.student.named_parameters():
        if k in update and digest[k]["norm"] >= floor:
            d = (p.detach() - p0[k]).flatten().double()[digest[k]["idx"].to(p.device)].cpu()
            mine.append(d / digest[k]["norm"]); ref.append(update[k].double() / digest[k]["norm"])
    a, b = torch.cat(mine), torch.cat(ref)
    rep["update_l2"] = float((a - b).norm() / b.norm())
    print("\nPARITY ifv step", name, {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        if k in ("ce", "pi", "G"):
            assert v < 1e-3, (k, v)
        elif k == "pa":
            assert v < 5e-3, (k, v)
        elif k.startswith("cwd"):
            assert v < 1e-2, (k, v)
        elif k.startswith("ifv"):
            assert v < 2e-2, (k, v)
    assert rep["logits_S"] < 3e-2
    assert rep["grad_norm"] < 0.6 and rep["grad_l2"] < 0.35 and rep["grad_cos"] > 0.93
    assert rep["update_l2"] < 0.35


# -------------------------------------------------------------------------------------------- graphs, repeatability, state, ranks
def _resnet18(batch, h, w, cfg, without=(), **extra):
    """NetModel with the ResNet18 student on the seeded weights, dropout masks, WGAN-GP alpha and batch of the golden cases; the
    argument fields named in `without` are removed, as in a namespace written before they existed."""
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**cfg)
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    torch.manual_seed(21)
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
GRAPH_EXTRA = dict(ifv=True, lambda_ifv=[0.0, 200.0, 0.0, 200.0, 200.0], cwd=True, overlap_streams=False)


def _terms(v):
    return [float(t) for t in v] if isinstance(v, list) else [float(v)]


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + _terms(m.ifv_G_loss) + [p.detach().clone() for p in m.student.parameters()] + \
        [b.detach().clone() for b in m.student.buffers()]


def _same(a, b):
    return len(a) == len(b) and all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


def _state(m):
    return [{k: v.clone() for k, v in mod.state_dict().items()} for mod in (m.student, m.D_model)] + \
        [m.G_solver.flat_m.clone(), m.D_solver.flat_m.clone()]


def _rewind(m, snap):
    with torch.no_grad():
        for mod, sd in zip((m.student, m.D_model), snap[:2]):
            cur = mod.state_dict()
            for k, v in sd.items():
                cur[k].copy_(v)                                           # in place: the captured graph reads these buffers
        m.G_solver.flat_m.copy_(snap[-2]); m.D_solver.flat_m.copy_(snap[-1])


def test_cuda_graph_replays_equal_eager_and_runs_repeat():
    """ResNet18 Pi + Pa + Ho + CWD on the logits + IFV at x2, x4 and the PSP features, 256x256 batch 2, overlap_streams off: two eager
    runs of three steps are bitwise equal, and three replays of the captured step, rewound to the starting state, equal them."""
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
    ifv = runs[0][0][2:7]
    assert ifv[0] == 0.0 and ifv[2] == 0.0 and all(ifv[i] > 0 for i in (1, 3, 4))          # zero weights log 0.0
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
    """IFV has no trainable state: the file keeps the keys of a run without it.  Three steps, a save, a load into a fresh CUDA-graph
    model and three more steps equal six uninterrupted steps bit for bit; a model without IFV loads the same file."""
    cfg = dict(pi=True, pa=True, ho=True, adv_type="hinge")
    extra = dict(ifv=True, lambda_ifv=[200.0, 0.0, 0.0, 0.0, 200.0], overlap_streams=False)
    want = []
    m = _resnet18(1, 256, 256, cfg, **extra)
    for k in range(6):
        m.optimize_parameters()
        if k == 2:
            m.save_training_state(str(tmp_path / "ifv.pth"), 3)
        if k >= 3:
            torch.cuda.synchronize()
            want.append(_dump(m))
    assert set(torch.load(str(tmp_path / "ifv.pth"), weights_only=False)) == BASE_KEYS
    del m
    m = _resnet18(1, 256, 256, cfg, **extra)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                   # captured
    assert m._graphs["captured"]
    assert m.load_training_state(str(tmp_path / "ifv.pth")) == 3
    for w in want:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)
    del m
    plain = _resnet18(1, 256, 256, cfg, overlap_streams=False)
    assert plain.load_training_state(str(tmp_path / "ifv.pth")) == 3


def test_defaults_launch_no_ifv_kernel(monkeypatch):
    """With make_args' defaults (ifv off, whatever lambda_ifv holds) no IFV kernel runs; G_solver's flat buffer and the state keys are
    those of a run without the IFV fields."""
    from structure_knowledge_distillation_b200 import ops

    def refuse(*a, **k):
        raise AssertionError("an IFV kernel ran with the term off")
    for fn in ("ifv_fwd", "ifv_bwd", "labels_nearest"):
        monkeypatch.setattr(ops, fn, refuse)
    cfg = dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    old = _resnet18(1, 256, 256, cfg, without=("ifv", "lambda_ifv"))
    layout = (old.G_solver.flat_p.numel(), [tuple(p.shape) for p in old.G_solver.params], set(old._extra_states()))
    del old
    for more in ({}, dict(lambda_ifv=[1.0] * 5)):
        m = _resnet18(1, 256, 256, cfg, **more)
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert m.ifv_G_loss is None and m.criterion_ifv == []
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
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, ifv=True,
                               lambda_ifv=[200.0, 0.0, 0.0, 0.0, 200.0]))
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
        if rank == 0:
            out.put(("ok", err, [float(v) for v in m.ifv_G_loss]))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_sums_the_shard_gradients():
    """ResNet18 with IFV at x1 and the PSP features over 2 NCCL ranks: the all-reduced flat gradient is the sum of the per-rank
    gradients.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29655, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY ifv world2", res)
    assert res[0] == "ok" and res[1] < 1e-6, res
