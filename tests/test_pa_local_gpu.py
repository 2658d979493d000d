"""Local pair-wise distillation on the H100: the csrc/pairwise_local.cu kernels against the float64 restatement (oracle/pa_local_port.py)
and, with a covering window, against the fully connected SIMT kernels; the memory of x1 at one node per pixel; NetModel steps against
tests/golden/pa_local.pt.gz; CUDA-graph replay, repeatability and two NCCL ranks."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _relf(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _nhwc(n, c, h, w, gen, pitch=None):
    """(N, C, H, W) view of a random NHWC buffer, the last c channels of a `pitch`-wide one when given (as the teacher's x4 is)."""
    p = pitch or c
    buf = torch.randn(n, h, w, p, generator=gen, device="cuda")
    return buf.permute(0, 3, 1, 2)[:, p - c:] if pitch else buf.permute(0, 3, 1, 2)


def _ref(S, T, ph, pw, k, d):
    """Loss and d loss / d S of the restatement in float64 (max pool (ph, pw), ceil mode)."""
    from oracle import pa_local_port as P
    sd = S.detach().double().contiguous().requires_grad_(True)
    ps = F.max_pool2d(sd, (ph, pw), (ph, pw), 0, ceil_mode=True)
    pt = F.max_pool2d(T.detach().double(), (ph, pw), (ph, pw), 0, ceil_mode=True)
    loss = P.local_affinity_loss(ps, pt, k, d)
    (g,) = torch.autograd.grad(loss, sd)
    return loss, g


def _mine(S, T, ph, pw, k, d, gscale=1.0):
    from structure_knowledge_distillation_b200 import functions as Fn
    Sg = S.detach().requires_grad_(True)
    loss = Fn.PairWiseLocalLoss.apply(Sg, T, ph, pw, k, d)
    (g,) = torch.autograd.grad(loss * gscale, Sg)
    return loss, g


# (N, C_S, C_T, H, W, ph, pw, k, d, student pitch, teacher pitch)
CASES = [
    (1, 8, 8, 1, 1, 1, 1, 3, 1, None, None),                  # one node
    (2, 19, 131, 7, 5, 1, 1, 15, 1, 20, None),                # grid smaller than the window; ESPNet widths, pitched student
    (2, 128, 512, 65, 129, 1, 1, 9, 1, None, None),           # PSP features at one node per pixel (batch 2)
    (1, 64, 256, 129, 257, 1, 1, 9, 2, None, None),           # x1 at one node per pixel
    (3, 131, 19, 30, 41, 2, 3, 5, 4, 132, 20),                # pooled 2x3 windows, both pitched, d = 4
    (2, 33, 70, 17, 23, 1, 1, 3, 8, None, 72),                # d = 8, teacher 2 floats into a 72-wide buffer
    (2, 512, 2048, 17, 31, 1, 1, 15, 2, None, 4096),          # ResNet18 x4 against the teacher's x4 slice of the PSP concat buffer
    (4, 1, 3, 9, 1, 1, 1, 5, 1, None, None),                  # one channel, n x 1
    (2, 6, 10, 1, 40, 1, 1, 9, 2, None, None),                # 1 x n
    (2, 96, 320, 45, 60, 1, 1, 15, 1, None, None),            # MobileNetV2's / ESPNet-C's 45x60 grid, k = 15
    (1, 24, 32, 90, 120, 3, 3, 5, 2, None, None),             # MobileNetV2's x1 pooled 3x3
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N%d_C%d-%d_%dx%d_p%dx%d_k%d_d%d" % c[:9])
def test_kernels_match_float64(case):
    """Loss and student gradient against the restatement's autograd in float64.  Bound: each affinity is an fp32 FMA sum of C products of
    normalised entries (|partial sums| <= 1 by Cauchy-Schwarz), so its absolute error is at most C * 2^-24 and typically sqrt(C) * 2^-24
    (1e-6 at C = 2048); independent random S and T give |E| ~ 1/sqrt(C) off the diagonal, so E and the loss carry a relative error of
    about C * 2^-24 <= 1.2e-4 in the worst case and 1e-5 typically; the backward's k^2-term fp32 sum adds k^2 * 2^-24 < 1.4e-5.  The
    loss's sum runs in double.  Asserted: loss 1e-4, gradient 2e-4."""
    n, cs, ct, H, W, ph, pw, k, d, sp, tp = case
    gen = torch.Generator(device="cuda").manual_seed(sum(case[:9]))
    S, T = _nhwc(n, cs, H, W, gen, sp), _nhwc(n, ct, H, W, gen, tp)
    loss, g = _mine(S, T, ph, pw, k, d, gscale=3.0)
    ref, gref = _ref(S, T, ph, pw, k, d)
    e_loss, e_grad = _relf(loss, ref), _rel(g.double(), 3.0 * gref)
    print("\nPARITY pa_local", case, "loss %.2e grad %.2e" % (e_loss, e_grad))
    if H * W == 1:                                               # one node: a_ii = 1 on both sides, the loss is rounding residue
        assert abs(float(loss)) < 1e-12 and float(g.abs().max()) < 1e-5
        return
    assert e_loss < 1e-4 and e_grad < 2e-4, (e_loss, e_grad)


@pytest.mark.parametrize("h, w, cs, ct", [(8, 8, 128, 512), (3, 7, 19, 131), (1, 8, 64, 256), (5, 1, 33, 70), (6, 5, 512, 2048)])
def test_covering_window_matches_global_simt_kernels(h, w, cs, ct):
    """d = 1 and a window covering the grid (k = 15 >= 2 max(h, w) - 1): loss and gradient equal those of the fully connected term's SIMT
    kernels (fewer than 1 024 nodes) to fp32 reordering, 2e-5 (loss) and 5e-5 (gradient)."""
    from structure_knowledge_distillation_b200 import functions as Fn
    gen = torch.Generator(device="cuda").manual_seed(h * 100 + w)
    S, T = _nhwc(2, cs, 2 * h, 3 * w, gen), _nhwc(2, ct, 2 * h, 3 * w, gen)
    loss, g = _mine(S, T, 2, 3, 15, 1)
    Sg = S.detach().requires_grad_(True)
    gl = Fn.PairWiseLoss.apply(Sg, T, 2, 3)
    (gg,) = torch.autograd.grad(gl, Sg)
    e_loss, e_grad = _relf(loss, gl), _rel(g, gg)
    print("\nPARITY pa_local vs global", (h, w, cs, ct), "loss %.2e grad %.2e" % (e_loss, e_grad))
    assert e_loss < 2e-5 and e_grad < 5e-5, (e_loss, e_grad)


def test_repeatable_bit_for_bit():
    """Two calls on the same inputs give identical losses and gradients (fixed-order reductions, no atomics)."""
    gen = torch.Generator(device="cuda").manual_seed(11)
    S, T = _nhwc(4, 128, 65, 129, gen), _nhwc(4, 512, 65, 129, gen)
    a, b = _mine(S, T, 1, 1, 9, 2), _mine(S, T, 1, 1, 9, 2)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_x1_one_node_per_pixel_memory():
    """x1 at 512x1024, batch 8, one node per pixel (129x257 = 33 153 nodes), k = 9: forward plus backward raises the peak allocation by
    under 1 GiB (E is 8 x 33 153 x 81 floats, 86 MB), where the fully connected term's E alone would be 8 x 33 153^2 floats, 35 GB."""
    from structure_knowledge_distillation_b200 import functions as Fn
    gen = torch.Generator(device="cuda").manual_seed(12)
    S, T = _nhwc(8, 64, 129, 257, gen), _nhwc(8, 256, 129, 257, gen)
    Sg = S.detach().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = Fn.PairWiseLocalLoss.apply(Sg, T, 1, 1, 9, 1)
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("\nPA_LOCAL x1 b8 k9 peak %.1f MB (global E would be %.1f GB)" % (peak / 2 ** 20, 8 * 33153 ** 2 * 4 / 1e9))
    assert torch.isfinite(loss) and peak < 2 ** 30


# -------------------------------------------------------------------------------------------- NetModel steps against the golden
def _args(spec, c, **extra):
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    return make_args(batch_size=spec["batch"], pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, student=spec["kind"],
                     lambda_pa=c.lambda_pa, pool_scale=c.pool_scale, pa_window=spec["window"], pa_dilation=spec["dilation"], **extra)


def _case_model(spec):
    from oracle import make_golden_pa_local as G, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    c = port.StepConfig(**spec["cfg"])
    teacher, student, D, images, labels, masks, alpha = G.case_inputs(spec)
    m = NetModel(_args(spec, c))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for drop, mk in zip(m.student.dropouts() if masks else [], masks):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = alpha.cuda()
    m.set_input((images, labels, None, None))
    return m, c


def _kept(digest):
    """Parameters whose golden gradient is not analytically vanishing: a norm of at least 1e-6 and 1e-3 x the median
    (tests/test_pa_levels_gpu.py's rule).  A BatchNorm shift whose output reaches a train-mode BatchNorm only through linear layers has a
    zero gradient; what the fp32 CPU and TF32 GPU steps leave there is cancellation residue of ~1e-6 (MobileNetV2's features.1 BN)."""
    norms = sorted(v["norm"] for v in digest.values())
    floor = max(1e-6, 1e-3 * norms[len(norms) // 2])
    return {k for k, v in digest.items() if v["norm"] >= floor}


def _samples(named, digest):
    """(mine, gold) rows of sampled values normalised by the golden's norm, and the worst relative norm error."""
    worst, mine_s, gold_s = 0.0, [], []
    kept = _kept(digest)
    for name, v in named:
        gd = digest.get(name)
        if name not in kept:
            continue
        a = v.detach().flatten().double()
        worst = max(worst, abs(float(a.norm()) - gd["norm"]) / gd["norm"])
        mine_s.append(a[gd["idx"].to(a.device)].cpu() / gd["norm"]); gold_s.append(gd["samples"].double() / gd["norm"])
    return torch.cat(mine_s), torch.cat(gold_s), worst


GOLDEN_NAMES = ["r18_psp_local9_pi_pa_ho_512_b1", "r18_x1_local9d2_psp_global_96x128_b2", "mobilenetv2_psp_local5_360x480_b1",
                "mobilenetv2_x1_local3d4_x4_global_360x480_b1", "espnet_c_psp_local15_360x480_b1", "espnet_c_x1_local7d2_psp_global_360x480_b1"]


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_step_matches_golden(name):
    """Losses, logits, sampled student gradients and the parameters after one SGD step against the fp32 CPU restatement, with
    tests/test_feature_kd_gpu.py's bounds: the task, Pi and total losses to 1e-3, each Pa term (read from the student's features,
    which carry the TF32 convolutions' rounding) to 5e-3; gradients agree in direction and norm, not to fp32, over the parameters whose
    gradient does not vanish analytically (_kept)."""
    from oracle import make_golden_pa_local as G
    from structure_knowledge_distillation_b200.utils.criterion import CriterionPairWiseLocal
    gold, spec = G.load()[name], G.GOLDEN_CASES[name]
    m, cfg = _case_model(spec)
    crits = m.criterion_pair_wise_for_interfeat
    crits = crits if isinstance(crits, list) else [crits]
    windows = spec["window"] if isinstance(spec["window"], list) else [spec["window"]]
    assert [isinstance(c, CriterionPairWiseLocal) for c in crits] == [w is not None for w in windows]
    p0 = {k: p.detach().clone() for k, p in m.student.named_parameters()}
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    rep = dict(ce=_relf(m.mc_G_loss, gold["ce"]), G=_relf(m.G_loss, gold["G"]), pi=_relf(m.pi_G_loss, gold["pi"]))
    mine, ref = (m.pa_G_loss, gold["pa"]) if isinstance(gold["pa"], list) else ([m.pa_G_loss], [gold["pa"]])
    assert len(mine) == len(ref)
    for ind, (a, b) in enumerate(zip(mine, ref)):
        if b == 0.0:
            assert a == 0.0 and isinstance(a, float)
        else:
            rep["pa%d" % ind] = _relf(a, b)
    rep["logits_S"] = _rel(m.preds_S[0][:, :, ::8, ::8].float().cpu(), gold["logits_S"])
    sm, sg, worst = _samples([(k, p.grad) for k, p in m.student.named_parameters()], gold["student_grads"])
    rep["grad_norm"], rep["grad_l2"] = worst, float((sm - sg).norm() / sg.norm())
    rep["grad_cos"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    m.G_solver.step()
    digest, update = gold["student_grads"], gold["student_update"]
    a_s, b_s, kept = [], [], _kept(digest)
    for k, p in m.student.named_parameters():
        if k in update and k in kept:
            dlt = (p.detach() - p0[k]).flatten().double()[digest[k]["idx"].to(p.device)].cpu()
            a_s.append(dlt / digest[k]["norm"]); b_s.append(update[k].double() / digest[k]["norm"])
    a, b = torch.cat(a_s), torch.cat(b_s)
    rep["update_l2"] = float((a - b).norm() / b.norm())
    print("\nPARITY pa_local step", name, {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        if k in ("ce", "pi", "G"):
            assert v < 1e-3, (k, v)
        elif k.startswith("pa"):
            assert v < 5e-3, (k, v)
    assert rep["logits_S"] < 3e-2
    assert rep["grad_norm"] < 0.6 and rep["grad_l2"] < 0.35 and rep["grad_cos"] > 0.93
    assert rep["update_l2"] < 0.35


# -------------------------------------------------------------------------------------------- graphs, repeatability, ranks
GRAPH_EXTRA = dict(lambda_pa=[0.5, 0.0, 0.5, 0.0, 0.5], pool_scale=[1.0 / 91, 0.5, 0.5, 0.5, 1.0 / 46],
                   pa_window=[9, None, None, None, 5], pa_dilation=[2, 1, 1, 1, 1], overlap_streams=False)


def _resnet18(batch, h, w, **extra):
    """NetModel (ResNet18, Pi + Pa + Ho wgan-gp) on the golden cases' seeded weights, dropout masks, alpha and batch."""
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", **extra))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for drop, mk in zip(m.student.dropouts(), cases.dropout_masks(student, batch, seed=2)):
        drop.injected = mk
    m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    return m


def _dump(m):
    pa = m.pa_G_loss if isinstance(m.pa_G_loss, list) else [m.pa_G_loss]
    return [float(m.G_loss), float(m.D_loss)] + [float(t) for t in pa] + \
        [p.detach().clone() for p in m.student.parameters()] + [b.detach().clone() for b in m.student.buffers()]


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


def test_cuda_graph_replays_equal_eager_and_runs_repeat():
    """ResNet18 Pi + Pa + Ho at 360x480, batch 2: x1 (91x121) local 9x9 at dilation 2 and the PSP features (46x61) local 5x5, both at one
    node per pixel, beside a fully connected x3.  Two eager runs of three steps are bitwise equal, and three replays of the captured
    step, rewound to the starting state, equal them."""
    runs = []
    for _ in range(2):
        m = _resnet18(2, 360, 480, **GRAPH_EXTRA)
        want = []
        for _ in range(3):
            m.optimize_parameters()
            torch.cuda.synchronize()
            want.append(_dump(m))
        runs.append(want)
        del m
    assert all(_same(a, b) for a, b in zip(*runs))
    pa = runs[0][0][2:7]                                              # x1, x2 (off), x3, x4 (off), PSP
    assert pa[1] == 0.0 and pa[3] == 0.0 and min(pa[0], pa[2], pa[4]) > 0.0, pa
    m = _resnet18(2, 360, 480, **GRAPH_EXTRA)
    snap = _state(m)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()
    assert m._graphs["captured"]
    _rewind(m, snap)
    for w in runs[0]:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)


def test_scalar_local_term_on_the_psp_features():
    """A scalar pa_window puts one local term on preds[-5]; pa_G_loss stays a scalar and print_info's format is unchanged."""
    from structure_knowledge_distillation_b200.utils.criterion import CriterionPairWiseLocal
    m = _resnet18(1, 256, 256, pool_scale=1.0 / 33, pa_window=7, pa_dilation=3)
    crit = m.criterion_pair_wise_for_interfeat
    assert isinstance(crit, CriterionPairWiseLocal) and (crit.feat_ind, crit.window, crit.dilation) == (-5, 7, 3)
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert not isinstance(m.pa_G_loss, list) and float(m.pa_G_loss) > 0.0
    from oracle import pa_local_port as P
    fS, fT = m.preds_S[-5].detach().double(), m.preds_T[-5].double()
    assert fS.shape[2:] == (33, 33)
    ref = P.pairwise_local_loss(fS, fT, 1.0 / 33, 7, 3)
    assert _relf(m.pa_G_loss, ref) < 1e-4


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
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world,
                               lambda_pa=[0.5, 0.0, 0.0, 0.0, 0.5], pool_scale=[1.0 / 91, 0.5, 0.5, 0.5, 1.0 / 46],
                               pa_window=[9, None, None, None, 15], pa_dilation=[2, 1, 1, 1, 1]))
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
            out.put(("ok", err, [float(v) for v in m.pa_G_loss]))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_step_sums_the_shard_gradients():
    """ResNet18 with local Pa at x1 and the PSP features over 2 NCCL ranks: the all-reduced flat gradient is the sum of the per-rank
    gradients.  Skipped with fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29653, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY pa_local world2", res)
    assert res[0] == "ok" and res[1] < 1e-6 and res[2][0] > 0.0 and res[2][4] > 0.0, res
