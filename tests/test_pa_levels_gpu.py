"""Multi-level pair-wise distillation (list-valued lambda_pa / pool_scale) on the H100: each level's loss and feature gradient
against float64, ResNet18 steps against the reference's multi-level loop (tests/golden/pa_levels.pt.gz, tools/pa_levels_oracle.py),
zero-weight levels, the other students against their float64 ports (resampled teacher levels included), CUDA-graph replay and two
NCCL ranks."""
import pytest
import torch

pytestmark = pytest.mark.gpu

LEVELS5 = dict(lambda_pa=[0.5, 0.0, 1.0, 2.0, 0.5], pool_scale=[0.5, 0.5, 0.5, 0.5, 0.5])


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _relf(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _resnet18(batch, h, w, cfg, graph=False, ho_alpha=True):
    """NetModel with the ResNet18 student on the seeded weights, dropout masks and batch of the golden cases."""
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    c = port.StepConfig(**cfg)
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    m = NetModel(make_args(batch_size=batch, pi=c.pi, pa=c.pa, ho=c.ho, adv_loss_type=c.adv_type, lambda_pi=c.lambda_pi,
                           lambda_pa=c.lambda_pa, lambda_d=c.lambda_d, lambda_gp=c.lambda_gp, pool_scale=c.pool_scale,
                           weight_decay=c.weight_decay, cuda_graph=graph))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    m.D_model.load_state_dict(D.state_dict())
    for drop, mk in zip(m.student.dropouts(), cases.dropout_masks(student, batch, seed=2)):
        drop.injected = mk
    if c.ho and c.adv_type == "wgan-gp" and ho_alpha:
        m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    return m, c


def test_each_resnet18_level_matches_float64():
    """Pa of each of the five ResNet18 levels on the features of a real forward (256x256, batch 2): loss and feature gradient against
    port.pairwise_loss in float64.  x1 at scale 1/65 is 65x65 = 4 225 nodes (the wgmma path); the teacher's x4 is its channel slice
    of the PSP concat buffer."""
    from oracle import port
    from structure_knowledge_distillation_b200 import functions as Fn
    scales = [1.0 / 65, 0.5, 0.25, 0.5, 0.125]
    m, _ = _resnet18(2, 256, 256, dict(pi=False, pa=True, ho=False, lambda_pa=[1.0] * 5, pool_scale=scales))
    m.forward()
    x4_T = m.preds_T[-4]
    assert x4_T.stride(3) == 2048 + 4 * 512 and x4_T.stride(1) == 1                  # pitched slice of the concat buffer
    assert tuple(m.preds_T[-1].shape[2:]) == (65, 65)
    rep = {}
    for ind, crit in enumerate(m.criterion_pair_wise_for_interfeat):
        i = crit.feat_ind
        assert i == -(ind + 1)
        fS = m.preds_S[i].detach().requires_grad_(True)
        fT = m.preds_T[i]
        S = list(m.preds_S); S[i] = fS
        loss = crit(S, m.preds_T)
        (g,) = torch.autograd.grad(loss, fS)
        sd = fS.detach().double().contiguous().requires_grad_(True)
        ref = port.pairwise_loss(sd, fT.double().contiguous(), scales[ind])
        (gref,) = torch.autograd.grad(ref, sd)
        h, w = fT.shape[2:]
        nodes = -(-h // int(h * scales[ind])) * -(-w // int(w * scales[ind]))
        rep[ind] = (nodes, _relf(loss, ref), _rel(g.double(), gref))
    print("\nPARITY pa_levels per level (nodes, loss rel, grad rel-L2)", rep)
    assert rep[0][0] >= Fn.PairWiseLoss.TCGEN05_MIN_NODES
    for ind, (nodes, e_loss, e_grad) in rep.items():
        # TF32 operands on the wgmma path (as tests/test_kernels_gpu.py bounds it); fp32 on the SIMT path
        assert e_loss < (1e-3 if nodes >= Fn.PairWiseLoss.TCGEN05_MIN_NODES else 1e-4), (ind, e_loss)
        assert e_grad < (1e-2 if nodes >= Fn.PairWiseLoss.TCGEN05_MIN_NODES else 1e-3), (ind, e_grad)


@pytest.mark.parametrize("name", ["levels5_pi_pa_96x128_b2", "level_x1_pi_pa_96x128_b2", "levels5_pi_pa_ho_wgangp_512_b1"])
def test_resnet18_step_matches_reference_golden(name):
    """NetModel list-mode steps against the reference's multi-level loop, within tests/test_step_gpu.py's bounds for these sizes."""
    from tools import pa_levels_oracle as O
    gold = O.load()[name]
    spec = O.GOLDEN_CASES[name]
    m, cfg = _resnet18(spec["batch"], spec["h"], spec["w"], spec["cfg"])
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    rep = dict(ce=_relf(m.mc_G_loss, gold["ce"]), pi=_relf(m.pi_G_loss, gold["pi"]), G=_relf(m.G_loss, gold["G"]))
    assert len(m.pa_G_loss) == len(gold["pa"])
    for ind, (mine, ref) in enumerate(zip(m.pa_G_loss, gold["pa"])):
        if ref == 0.0:
            assert mine == 0.0 and isinstance(mine, float)
        else:
            rep["pa%d" % ind] = _relf(mine, ref)
    rep["logits_S"] = _rel(m.preds_S[0][:, :, ::8, ::8].float().cpu(), gold["logits_S"])
    rep["logits_T"] = _rel(m.preds_T[0][:, :, ::8, ::8].float().cpu(), gold["logits_T"])
    rep["feat_T"] = max(_relf(m.preds_T[-(ind + 1)].norm(), v) for ind, v in enumerate(gold["feat_norms_T"]))
    worst, samp_mine, samp_gold = 0.0, [], []
    for pname, p in m.student.named_parameters():
        gd = gold["student_grads"].get(pname)
        if gd is None or gd["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        worst = max(worst, abs(float(mine.norm()) - gd["norm"]) / gd["norm"])
        samp_mine.append(mine[gd["idx"].to(mine.device)].cpu() / gd["norm"]); samp_gold.append(gd["samples"].double() / gd["norm"])
    sm, sg = torch.cat(samp_mine), torch.cat(samp_gold)
    rep["worst_student_grad_norm_rel"] = worst
    rep["student_grad_samples_rel_l2"] = float((sm - sg).norm() / sg.norm())
    rep["student_grad_samples_cosine"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    if cfg.ho:
        m.G_solver.step()
        m.discriminator_backward()
        rep["D"] = _relf(m.D_loss, gold["D"])
        top = max(g["norm"] for g in gold["D_grads"].values())
        rep["worst_D_grad_norm_rel"] = max(abs(float(p.grad.double().norm()) - gold["D_grads"][k]["norm"]) /
                                           max(gold["D_grads"][k]["norm"], 1e-3 * top)
                                           for k, p in m.D_model.named_parameters() if k in gold["D_grads"] and p.grad is not None)
    print("\nPARITY pa_levels step", name, {k: "%.2e" % v for k, v in rep.items()})
    for k, v in rep.items():
        if k in ("ce", "pi", "G", "D"):
            assert v < 1e-3, (k, v)
        elif k.startswith("pa"):
            assert v < 5e-3, (k, v)          # Pa of a random-init student at batch 1-2 under TF32 (tests/test_step_gpu.py)
    assert rep["logits_T"] < 2e-3 and rep["logits_S"] < 3e-2 and rep["feat_T"] < 2e-3
    assert rep["worst_student_grad_norm_rel"] < 0.6
    assert rep["student_grad_samples_rel_l2"] < 0.35 and rep["student_grad_samples_cosine"] > 0.93
    if cfg.ho:
        assert rep["worst_D_grad_norm_rel"] < 0.3


def test_zero_weight_levels_launch_nothing_and_log_zero():
    """Levels with lambda 0 cost no kernel: [l, 0, 0, 0, 0] launches exactly what the one-entry list [l] does, and logs 0.0 for the
    four others; a level whose pooling window comes out empty raises ValueError naming it at the first forward."""
    from structure_knowledge_distillation_b200._cabi import lib
    L = lib()
    counts, first = [], []
    for lam, scale in (([0.5], [0.25]), ([0.5, 0.0, 0.0, 0.0, 0.0], [0.25, 0.5, 0.5, 0.5, 0.5])):
        m, _ = _resnet18(2, 96, 128, dict(pi=True, pa=True, ho=False, lambda_pa=lam, pool_scale=scale))
        m.forward(); m.G_solver.zero_grad(); m.student_backward()                  # warm: workspaces, kernels loaded
        torch.cuda.synchronize()
        l0 = L.skd_kernel_launches()
        m.forward(); m.G_solver.zero_grad(); m.student_backward()
        torch.cuda.synchronize()
        counts.append(L.skd_kernel_launches() - l0)
        first.append(float(m.pa_G_loss[0]))
        assert all(v == 0.0 and isinstance(v, float) for v in m.pa_G_loss[1:])
        del m
    print("\nPA_LEVELS launches per forward + backward: one level %d, one level + four zero-weight levels %d" % tuple(counts))
    assert counts[0] == counts[1] and first[0] == first[1]
    m, _ = _resnet18(2, 96, 128, dict(pi=False, pa=True, ho=False, lambda_pa=[0.5, 0.5], pool_scale=[0.5, 0.05]))
    m.forward(); m.G_solver.zero_grad()
    with pytest.raises(ValueError, match=r"pair-wise level 1 \(preds\[-2\]"):
        m.student_backward()


def _student_case(kind):
    """(NetModel, float64 port student, teacher, batch) for a non-ResNet18 student at 360x480, batch 2, Pi + five Pa levels."""
    from oracle import cases, espnet_full_port, espnet_port, mobilenet_port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    teacher, _, _ = cases.build_models(seed=0, with_D=False)
    ref = {"espnet_c": espnet_port, "espnet": espnet_full_port, "mobilenetv2": mobilenet_port}[kind].build_student(7)
    m = NetModel(make_args(batch_size=2, pi=True, pa=True, ho=False, student=kind, **LEVELS5))
    m.student.load_state_dict(ref.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    if kind == "mobilenetv2":
        for d, mk in zip(m.student.dropouts(), cases.dropout_masks(ref, 2, seed=2)):
            d.injected = mk
        for d, mk in zip(ref.dropouts(), cases.dropout_masks(ref, 2, seed=2)):
            d.injected = mk.cuda()
    return m, ref, teacher


@pytest.mark.parametrize("kind", ["espnet_c", "espnet", "mobilenetv2"])
def test_other_students_match_float64_port(kind):
    """ESPNet-C, ESPNet and MobileNetV2 list-mode steps (five levels at scale 0.5, x2's weight 0) against the multi-level loop over
    their oracle ports in float64 on the GPU.  Their levels sit on other grids than the teacher's (ESPNet's b1 at 1/2, MobileNetV2's
    maps by rounding): the teacher's are resampled onto them."""
    from oracle import port
    from tools import pa_levels_oracle as O
    m, ref, teacher = _student_case(kind)
    images, labels = port.synthetic_batch(2, 360, 480, seed=1)
    m.set_input((images, labels, None, None))
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    tf = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        refd, td = ref.cuda().double(), teacher.cuda().double()
        cfg = port.StepConfig(pi=True, pa=True, ho=False, **LEVELS5)
        out = O.distill_step(kind, td, refd, None, images.cuda().double(), labels.cuda(), cfg)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf
    grids = {ind: (tuple(out["preds_T"][-(ind + 1)].shape[2:]), tuple(m.preds_T[-(ind + 1)].shape[2:])) for ind in range(5)}
    rep = dict(ce=_relf(m.mc_G_loss, out["ce"]), pi=_relf(m.pi_G_loss, out["pi"]), G=_relf(m.G_loss, out["G"]))
    for ind, (mine, r) in enumerate(zip(m.pa_G_loss, out["pa"])):
        if r == 0.0:
            assert mine == 0.0
        else:
            rep["pa%d" % ind] = _relf(mine, r)
    norms = {k: float(p.grad.norm()) for k, p in refd.named_parameters() if p.grad is not None}
    med = sorted(norms.values())[len(norms) // 2]
    worst, wn, dots, nm, nr = 0.0, None, 0.0, 0.0, 0.0
    mine_p = dict(m.student.named_parameters())
    for k, p in refd.named_parameters():
        if p.grad is None or norms[k] < 1e-3 * med:                 # analytically vanishing gradients: cancellation residue
            continue
        a, b = mine_p[k].grad.detach().double().flatten(), p.grad.flatten()
        e = float((a - b).norm() / b.norm())
        if e > worst:
            worst, wn = e, k
        dots += float((a * b).sum()) / norms[k] ** 2; nm += float(a.norm()) ** 2 / norms[k] ** 2; nr += 1.0
    rep["worst_student_grad_rel_l2"] = (worst, wn)
    rep["student_grad_cosine"] = dots / (nm * nr) ** 0.5
    print("\nPARITY pa_levels", kind, "grids (port, ours)", grids, rep)
    for ind in range(5):                                            # the teacher's weighted levels on the student's grids
        assert grids[ind][0] == grids[ind][1], (ind, grids[ind])
        if LEVELS5["lambda_pa"][ind] != 0.0:
            assert grids[ind][1] == tuple(m.preds_S[-(ind + 1)].shape[2:]), (ind, grids[ind])
    for k, v in rep.items():
        if k in ("ce", "pi", "G"):
            assert v < 1e-3, (k, v)
        elif k.startswith("pa"):
            assert v < 5e-3, (k, v)
    assert rep["student_grad_cosine"] > 0.999, rep
    assert worst < 5e-2, rep["worst_student_grad_rel_l2"]


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + [float(v) for v in m.pa_G_loss] + \
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


def test_cuda_graph_replays_equal_eager_steps():
    """ResNet18, Pi + five Pa levels (one at weight 0) + Ho wgan-gp, 360x480 batch 2: three replays of the captured step, rewound to
    the starting state after the capture, equal three eager steps from that state bit for bit."""
    cfg = dict(pi=True, pa=True, ho=True, adv_type="wgan-gp", **LEVELS5)
    m, _ = _resnet18(2, 360, 480, cfg)
    want = []
    for _ in range(3):
        m.optimize_parameters()
        torch.cuda.synchronize()
        want.append(_dump(m))
    del m
    m, _ = _resnet18(2, 360, 480, cfg)
    snap = _state(m)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                     # eager warm-up, capture
    assert m._graphs["captured"]
    _rewind(m, snap)
    for w in want:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), w)


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
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, **LEVELS5))
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


def test_two_rank_list_mode_step_sums_the_shard_gradients():
    """ResNet18 list-mode step over 2 NCCL ranks: the all-reduced student gradient is the sum of the per-rank gradients.  Skipped with
    fewer than two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29641, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY pa_levels_world2", res)
    assert res[0] == "ok", res
