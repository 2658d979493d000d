"""H100: the OHEM cross entropy kernels (csrc/ohem.cu, the OHEM row kernel of csrc/losses.cu) and criteria against the
restatement in tools/ohem_oracle.py and the golden fixture made by the UNMODIFIED reference classes (tests/golden/ohem.pt),
and NetModel(ohem=True) against a golden step made by the reference modules driven with CriterionOhemDSN."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "ohem.pt"), weights_only=False)


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _layout(t, kind):
    """(N, C, h, w) CPU tensor -> CUDA tensor in NCHW, NHWC or 20-channel pitched NHWC storage."""
    from structure_knowledge_distillation_b200 import ops
    if t is None:
        return None
    t = t.cuda()
    if kind == "nchw":
        return t.contiguous()
    if kind == "nhwc":
        return t.contiguous(memory_format=torch.channels_last)
    n, c, h, w = t.shape
    buf = ops.empty_nhwc(n, c, h, w, t.device, pitch=c + 1)
    buf.copy_(t)
    return buf


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("name", ["dsn_65x129_512x1024", "dsn_zero_column_360x480", "dsn_half_way_36x44", "standalone_97x131_f4"])
def test_grid_sample_matches_restatement(name):
    from structure_knowledge_distillation_b200 import ops
    from tools import ohem_oracle as O
    c = O.OHEM_CASES[name]
    preds, labels = O.ohem_inputs(name)
    H, W = labels.shape[1:]
    up = preds[0] if c.get("standalone") else F.interpolate(preds[0], size=(H, W), mode="bilinear", align_corners=True)
    ref_pred, ref_lab = O.ohem_grid(torch.softmax(up, 1).numpy(), labels.numpy(), c["factor"])
    for kind in ("nchw", "nhwc", "pitched"):
        pred, glab, nvalid = ops.ohem_grid_sample(_layout(preds[0], kind), labels.cuda(), c["factor"], 255, want_labels=True)
        pred, glab = pred.cpu().numpy(), glab.cpu().numpy()
        assert pred.shape == ref_pred.shape and np.array_equal(glab, ref_lab), (name, kind)
        fin = np.isfinite(ref_pred)
        assert np.array_equal(np.isfinite(pred), fin) and int(nvalid) == int(fin.sum())
        err = np.abs(pred[fin].astype(np.float64) - ref_pred[fin]) / np.maximum(ref_pred[fin], 1e-6)
        assert err.max() < 2e-5, (name, kind, err.max())
        if name == "dsn_zero_column_360x480":
            assert (pred[:, :, -1] == 0).all() and (glab[:, :, -1] == 0).all()


@pytest.mark.parametrize("n", [1, 7, 1000, 65537, 1 << 20, 4 << 20])
def test_radix_select_equals_kthvalue(n):
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    v = torch.rand(n, device="cuda", generator=g)
    v[: n // 3] = torch.round(v[: n // 3] * 16) / 16                         # heavy duplicates
    v[torch.rand(n, device="cuda", generator=g) < 0.05] = 0.0
    v[torch.rand(n, device="cuda", generator=g) < 0.1] = float("inf")        # ignored points sort last
    nv = int(torch.isfinite(v).sum())
    nvalid = torch.tensor([nv], device="cuda", dtype=torch.int32)
    valid = v[torch.isfinite(v)]
    for mk in sorted({1, 2, max(1, nv // 3), max(1, nv - 1)}):
        if mk >= nv:
            continue
        thr = ops.ohem_threshold(v, nvalid, mk, -1.0)                          # thresh below every value: the bare order statistic
        ref = torch.kthvalue(valid.cpu(), mk).values
        assert float(thr) == float(ref), (n, mk, float(thr), float(ref))
        thr2 = ops.ohem_threshold(v, nvalid, mk, 0.5)
        assert float(thr2) == max(0.5, float(ref))
    assert float(ops.ohem_threshold(v, nvalid, nv, 0.7)) == 1.0               # min_kept >= valid
    if nv > 0:
        assert float(ops.ohem_threshold(v, nvalid, 0, 0.7)) == np.float32(0.7)   # min_kept 0


# ------------------------------------------------------------------------------------------------ criteria
def _run_criterion(name, kind):
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN, OhemCrossEntropy2d
    from tools import ohem_oracle as O
    c = O.OHEM_CASES[name]
    preds, labels = O.ohem_inputs(name)
    xs = [None if t is None else _layout(t, kind).requires_grad_(True) for t in preds]
    if c.get("standalone"):
        crit = OhemCrossEntropy2d(255, c["thresh"], c["min_kept"], c["factor"])
        loss = crit(xs[0], labels.cuda())
    else:
        crit = CriterionOhemDSN(255, c["thresh"], c["min_kept"])
        loss = crit(xs, labels.cuda())
    loss.backward()
    return loss, crit, xs


@pytest.mark.parametrize("kind", ["nchw", "nhwc", "pitched"])
def test_criteria_match_reference_golden(kind):
    from oracle import cases
    from tools import ohem_oracle as O
    gold = _gold()["criterion"]
    for name in O.OHEM_CASES:
        G = gold[name]
        loss, crit, xs = _run_criterion(name, kind)
        thr, kept = float(crit.last_threshold), float(crit.last_kept)
        report = dict(loss=_rel(loss, G["loss"]), thr=_rel(thr, G["threshold"]), kept=_rel(kept, G["kept"]))
        for key, x in (("d_l0", xs[0]), ("d_l1", xs[1])):
            if key in G:
                a, b = cases.at_stored(x.grad.detach().cpu(), G[key])
                report[key] = float((a - b).norm() / b.norm())
        print("\nPARITY ohem", name, kind, {k: "%.2e" % v for k, v in report.items()})
        assert report["loss"] <= 1e-4 and report["thr"] <= 1e-6 and report["kept"] <= 1e-4, (name, report)
        assert all(report[k] <= 2e-4 for k in ("d_l0", "d_l1") if k in report), (name, report)


def test_all_ignored_gives_nan_loss_and_zero_gradients():
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN, OhemCrossEntropy2d
    l0 = torch.randn(2, 19, 9, 9, device="cuda", requires_grad=True)
    l1 = torch.randn(2, 19, 9, 9, device="cuda", requires_grad=True)
    labels = torch.full((2, 64, 64), 255, device="cuda", dtype=torch.int64)
    crit = CriterionOhemDSN()
    loss = crit([l0, l1], labels)
    loss.backward()
    assert torch.isnan(loss) and float(crit.last_kept) == 0
    assert torch.equal(l0.grad, torch.zeros_like(l0)) and torch.equal(l1.grad, torch.zeros_like(l1))
    # head 0 empty only (threshold below every probability): NaN loss, zero head-0 gradient, finite head-1 gradient
    p = torch.randn(1, 19, 32, 32, device="cuda", requires_grad=True)
    lab = torch.randint(0, 19, (1, 32, 32), device="cuda")
    c2 = OhemCrossEntropy2d(thresh=0.0, min_kept=0, factor=4)
    out = c2(p, lab)
    out.backward()
    assert torch.isnan(out) and float(c2.last_kept) == 0 and torch.equal(p.grad, torch.zeros_like(p))


def test_standalone_width_limit_is_explicit():
    """OhemCrossEntropy2d at label resolution: 1 483 columns with 19 classes run, one more raises (documented limit)."""
    from structure_knowledge_distillation_b200.utils.criterion import OhemCrossEntropy2d
    for W, ok in ((1483, True), (1484, False)):
        p = torch.randn(1, 19, 8, W, device="cuda", requires_grad=True)
        lab = torch.randint(0, 19, (1, 8, W), device="cuda")
        crit = OhemCrossEntropy2d(factor=4)
        if ok:
            crit(p, lab).backward()
            assert torch.isfinite(p.grad).all() and float(crit.last_kept) > 0
        else:
            with pytest.raises(RuntimeError, match="source width too large"):
                crit(p, lab)


# ------------------------------------------------------------------------------------------------ step
def _ohem_model(cuda_graph=False):
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    from tools import ohem_oracle as O
    s = O.OHEM_STEP
    cfg = port.StepConfig(**s["cfg"])
    teacher, student, _ = cases.build_models(seed=0, with_D=False)
    torch.manual_seed(0)
    m = NetModel(make_args(batch_size=s["batch"], pi=cfg.pi, pa=cfg.pa, ho=cfg.ho, pool_scale=cfg.pool_scale, ohem=True,
                           ohem_thres=s["thresh"], ohem_keep=s["min_kept"]))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict())
    images, labels = port.synthetic_batch(s["batch"], s["h"], s["w"], seed=1)
    for drop, mk in zip(m.student.dropouts(), cases.dropout_masks(student, s["batch"], seed=2)):
        drop.injected = mk
    m.set_input((images, labels, None, None))
    return m, (images, labels)


def test_netmodel_ohem_step_matches_reference_golden():
    """Tolerances of tests/test_step_gpu.py for the small cases."""
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN
    gold = _gold()["step"]
    m, _ = _ohem_model()
    assert isinstance(m.criterion, CriterionOhemDSN)
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    report = {k: _rel(v, gold[k]) for k, v in dict(ce=m.mc_G_loss, pi=m.pi_G_loss, pa=m.pa_G_loss, G=m.G_loss).items()}
    lg = m.preds_S[0][:, :, ::8, ::8].float().cpu()
    report["logits_S"] = float((lg - gold["logits_S"]).norm() / gold["logits_S"].norm())
    worst, sm, sg = 0.0, [], []
    for pname, p in m.student.named_parameters():
        g = gold["student_grads"].get(pname)
        if g is None or g["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        worst = max(worst, abs(float(mine.norm()) - g["norm"]) / g["norm"])
        sm.append(mine[g["idx"].to(mine.device)].cpu() / g["norm"]); sg.append(g["samples"].double() / g["norm"])
    sm, sg = torch.cat(sm), torch.cat(sg)
    report["worst_grad_norm"] = worst
    report["grad_samples_rel_l2"] = float((sm - sg).norm() / sg.norm())
    report["grad_samples_cosine"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    thr, kept = float(m.criterion.last_threshold), float(m.criterion.last_kept)
    report["threshold"], report["kept"] = _rel(thr, gold["threshold"]), _rel(kept, gold["kept"])
    print("\nPARITY ohem_step", {k: "%.2e" % v for k, v in report.items()}, "threshold", thr, "kept", kept, "of", gold["valid"])
    # the mask is active: about half of the valid pixels are dropped, at nearly the reference's threshold and count (the student's
    # TF32 logits move p[label], and with it the order statistic and the pixels next to it, by ~1e-3)
    assert thr < 0.7 and kept < 0.7 * gold["valid"]
    assert report["threshold"] < 2e-2 and report["kept"] < 2e-2, report
    for k in ("ce", "pi", "G"):
        assert report[k] < 1e-3, (k, report[k])
    assert report["pa"] < 5e-3 and report["logits_S"] < 3e-2
    assert worst < 0.6 and report["grad_samples_rel_l2"] < 0.35 and report["grad_samples_cosine"] > 0.93, report


def _snapshot(m):
    return [{k: v.clone() for k, v in m.student.state_dict().items()}, m.G_solver.flat_m.clone()]


def _restore(m, snap):
    with torch.no_grad():
        cur = m.student.state_dict()
        for k, v in snap[0].items():
            cur[k].copy_(v)                                           # in place: a captured graph keeps reading these buffers
        m.G_solver.flat_m.copy_(snap[1])


def test_ohem_step_cuda_graph_replays_and_determinism():
    m, (images, labels) = _ohem_model()
    valid = int((labels != 255).sum())
    snap = _snapshot(m)

    def record(model):
        return (float(model.G_loss), float(model.mc_G_loss), float(model.criterion.last_threshold), float(model.criterion.last_kept))

    def eager():
        _restore(m, snap)
        m.set_input((images, labels, None, None))
        m.optimize_parameters()
        return record(m), m.G_solver.flat_p.clone()

    (a, pa), (b, pb) = eager(), eager()
    assert a == b and torch.equal(pa, pb), "two runs of the step differ"
    # five eager steps from the snapshot, then the same five steps as CUDA-graph replays: the student changes every step, so the
    # threshold (the order statistic of its probabilities) does too, and a replay must recompute it inside the graph
    _restore(m, snap)
    ref = []
    for _ in range(5):
        m.set_input((images, labels, None, None))
        m.optimize_parameters()
        ref.append(record(m))
    g, _ = _ohem_model()
    g.student.load_state_dict(m.student.state_dict())
    g.enable_cuda_graphs(warmup=2)
    for _ in range(3):                                                    # 2 eager + capture
        g.set_input((images, labels, None, None))
        g.optimize_parameters()
    assert g._graphs["captured"]
    _restore(g, snap)
    got = []
    for _ in range(5):
        g.set_input((images, labels, None, None))
        g.optimize_parameters()
        got.append(record(g))
    print("\nPARITY ohem_graph eager", ref, "replayed", got)
    assert len({r[2] for r in ref}) == 5 and all(0 < r[3] < 0.7 * valid for r in ref), ref
    for x, y in zip(ref, got):
        assert _rel(y[0], x[0]) < 1e-6 and _rel(y[1], x[1]) < 1e-6 and y[2] == x[2] and y[3] == x[3], (x, y)


def _ddp_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port as oport
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        # one 96x128 image per rank: 12 x 16 grid points, min_kept // 64 = 96 puts the threshold near their median
        keep = 96 * 64
        m = NetModel(make_args(batch_size=1, pi=True, pa=False, ho=False, ohem=True, ohem_thres=0.0, ohem_keep=keep, gpu_num=world))
        images, labels = oport.synthetic_batch(1, 96, 128, seed=7 + rank)                  # each rank its own shard
        m.set_input((images, labels, None, None))
        m._student_phase()
        # the single-process criterion on this rank's shard (the logits this rank's step produced)
        single = CriterionOhemDSN(thresh=0.0, min_kept=keep)
        preds = [t.detach() for t in m.preds_S[:2]]
        loss = single(preds, m.labels)
        assert float(m.mc_G_loss) == float(loss), (rank, float(m.mc_G_loss), float(loss))
        assert float(m.criterion.last_threshold) == float(single.last_threshold)
        assert float(m.criterion.last_kept) == float(single.last_kept) < float((m.labels != 255).sum())
        # the shards give different thresholds, and neither is the threshold of the whole two-image batch
        thr = m.criterion.last_threshold.reshape(1).clone()
        thrs = [torch.empty_like(thr) for _ in range(world)]
        dist.all_gather(thrs, thr)
        both = []
        for t in (preds[0], preds[1], m.labels):
            parts = [torch.empty_like(t.contiguous()) for _ in range(world)]
            dist.all_gather(parts, t.contiguous())
            both.append(torch.cat(parts))
        whole = CriterionOhemDSN(thresh=0.0, min_kept=keep * world)
        whole(both[:2], both[2])
        assert float(thrs[0]) != float(thrs[1]), [float(t) for t in thrs]
        assert all(float(t) != float(whole.last_threshold) for t in thrs), ([float(t) for t in thrs], float(whole.last_threshold))
        if rank == 0:
            out.put(("ok",))
    except Exception as e:                                                # noqa: BLE001
        out.put((repr(e),))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_ohem_loss_is_per_shard():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29613, q), nprocs=2, join=True)
    res = q.get(timeout=10)
    assert res[0] == "ok", res
