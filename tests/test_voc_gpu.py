"""PASCAL VOC on the H100: the augmentation kernel and test preprocessing against the UNMODIFIED reference loaders
(tests/golden/voc_dataset.pt.gz), the loss kernels at 21 classes against torch, the 21-class distillation step of each student against
the reference (tests/golden/steps_voc.pt, ResNet18) or the float64 ports (ESPNet-C, ESPNet), CUDA-graph replay, OHEM, evaluation
through a VOC loader, and the two-rank step."""
import gzip
import os
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C21 = 21


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _gold_loader():
    return torch.load(gzip.open(os.path.join(ROOT, "tests", "golden", "voc_dataset.pt.gz")), weights_only=False)


# ------------------------------------------------------------------------------------------------ loaders
def test_augment_kernel_matches_reference_voc_loader_bit_exact():
    from structure_knowledge_distillation_b200.dataset import VOC_SCALES, DeviceAugment, draw_augmentation
    gold = _gold_loader()
    total = 0
    for case in gold["cases"]:
        img, lab = case["raw_image"], case["raw_label"]
        n = len(case["items"])
        random.seed(case["seed"]); np.random.seed(case["seed"])
        augs = [draw_augmentation(img.shape[0], img.shape[1], case["crop"], case["scale"], case["mirror"], VOC_SCALES) for _ in range(n)]
        for dtype in (torch.float32, torch.int64):
            aug = DeviceAugment(case["crop"], case["mean"], 255, label_dtype=dtype, voc=True)
            out_i, out_l = aug([img] * n, [lab] * n, torch.tensor(augs, dtype=torch.float64))
            torch.cuda.synchronize()
            for k, (ri, rl) in enumerate(case["items"]):
                assert torch.equal(out_i[k].cpu(), ri), (case["name"], k)
                assert torch.equal(out_l[k].cpu().float(), rl), (case["name"], k)
                total += 1
    print("\nPARITY voc_dataset_golden %d samples bit-exact vs the reference VOCDataSet (cv2 %s)" % (total // 2, gold["cv2"]))


def test_test_preprocess_matches_reference_voc_test_set_bit_exact():
    from structure_knowledge_distillation_b200.dataset import DeviceTestPreprocess, numpy_mean
    for case in _gold_loader()["test_cases"]:
        out = DeviceTestPreprocess(case["crop"], numpy_mean(case["mean"]))([case["raw_image"]])
        assert torch.equal(out[0].cpu(), case["image"]), case["name"]


def test_cityscapes_entry_point_is_the_generic_kernel_with_the_id_table():
    """skd_cs_augment_batch (float32 mean, Cityscapes table) and skd_augment_batch with that table and the mean rounded to float32
    write the same bits; with no table the raw labels pass through."""
    import ctypes
    from structure_knowledge_distillation_b200 import _cabi
    from structure_knowledge_distillation_b200.dataset import Augmentation, DeviceAugment, cityscapes_id_tables
    from structure_knowledge_distillation_b200.dataset.datasets import _Sample
    g = np.random.default_rng(9)
    img = torch.from_numpy(g.integers(0, 256, (70, 90, 3), dtype=np.uint8)).cuda()
    lab = torch.from_numpy(g.integers(0, 256, (70, 90), dtype=np.uint8)).cuda()
    mean = np.array((104.00698793, 116.66876762, 122.67891434), np.float32)
    augs = torch.tensor([Augmentation(3, 1.0, 70, 90, 5, 7, -1), Augmentation(-1, 1.0, 70, 90, 0, 3, 1)], dtype=torch.float64)
    new_i, new_l = DeviceAugment((48, 64), mean)([img] * 2, [lab] * 2, augs)
    arr = (_Sample * 2)()
    for i, a in enumerate(augs.tolist()):
        s = arr[i]
        s.image, s.label, s.src_h, s.src_w = img.data_ptr(), lab.data_ptr(), 70, 90
        s.f_scale = a[1] if a[0] >= 0 else 0.0
        s.scaled_h, s.scaled_w, s.h_off, s.w_off, s.flip = int(a[2]), int(a[3]), int(a[4]), int(a[5]), int(a[6])
    old_i, old_l = torch.empty_like(new_i), torch.empty_like(new_l)
    m32 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    _cabi.lib().skd_cs_augment_batch(2, ctypes.cast(arr, ctypes.c_void_p), 48, 64, ctypes.cast(m32, ctypes.c_void_p), 255,
                                     old_i.data_ptr(), old_l.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(old_i, new_i) and torch.equal(old_l, new_l)
    raw_i, raw_l = DeviceAugment((48, 64), mean, voc=True)([img] * 2, [lab] * 2, augs)
    assert torch.equal(raw_i, new_i)
    to_train = torch.from_numpy(cityscapes_id_tables()[0].astype(np.int64)).cuda()
    assert torch.equal(to_train[raw_l], new_l)


def test_argument_errors_name_the_entry_point_called():
    """Both entry points share one implementation; a bad sample is reported under the name of the one the caller used."""
    import ctypes
    from structure_knowledge_distillation_b200 import _cabi
    from structure_knowledge_distillation_b200.dataset.datasets import _Sample
    L = _cabi.lib()
    arr = (_Sample * 1)()                                                  # NULL image / label: rejected before any launch
    out = torch.empty(1, 3, 8, 8, device="cuda"); lab = torch.empty(1, 8, 8, dtype=torch.int64, device="cuda")
    m32, m64 = (ctypes.c_float * 3)(0, 0, 0), (ctypes.c_double * 3)(0, 0, 0)
    with pytest.raises(RuntimeError, match="skd_cs_augment_batch"):
        L.skd_cs_augment_batch(1, ctypes.cast(arr, ctypes.c_void_p), 8, 8, ctypes.cast(m32, ctypes.c_void_p), 255, out.data_ptr(),
                               lab.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)
    assert L.last_error().startswith("skd_cs_augment_batch")
    with pytest.raises(RuntimeError, match="skd_augment_batch"):
        L.skd_augment_batch(1, ctypes.cast(arr, ctypes.c_void_p), 8, 8, ctypes.cast(m64, ctypes.c_void_p), None, 255, out.data_ptr(),
                            lab.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)
    assert L.last_error().startswith("skd_augment_batch")


def test_voc_loaders_end_to_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from oracle import voc_port as vp
    from structure_knowledge_distillation_b200.dataset import CSDataLoader, VOCDataSet, VOCDataTestSet
    (tmp_path / "JPEGImages").mkdir(); (tmp_path / "SegmentationClassAug").mkdir()
    rng = np.random.default_rng(3)
    raws = []
    with open(tmp_path / "train.txt", "w") as f:
        for i in range(4):
            img = rng.integers(0, 256, (75, 100, 3), dtype=np.uint8); lab = rng.integers(0, 21, (75, 100), dtype=np.uint8)
            cv2.imwrite(str(tmp_path / "JPEGImages" / ("n%d.jpg" % i)), img)
            cv2.imwrite(str(tmp_path / "SegmentationClassAug" / ("n%d.png" % i)), lab)
            f.write("n%d\n" % i)
            raws.append((cv2.imread(str(tmp_path / "JPEGImages" / ("n%d.jpg" % i))), lab))
    ds = VOCDataSet(str(tmp_path), str(tmp_path / "train.txt"), crop_size=(64, 80))
    random.seed(5); np.random.seed(5)
    batches = list(CSDataLoader(ds, batch_size=2))
    random.seed(5); np.random.seed(5)
    k = 0
    for images, labels, sizes, names in batches:
        assert images.is_cuda and labels.is_cuda and labels.dtype == torch.int64 and tuple(images.shape) == (2, 3, 64, 80)
        for j in range(2):
            wi, wl, _ = vp.voc_getitem(raws[k][0], raws[k][1], (64, 80), (128, 128, 128))
            assert np.array_equal(images[j].cpu().numpy(), wi) and np.array_equal(labels[j].cpu().numpy().astype(np.float32), wl)
            assert names[j] == "n%d" % k and tuple(int(v) for v in sizes[j]) == (75, 100, 3)
            k += 1
    assert k == 4
    mean = (104.00698793, 116.66876762, 122.67891434)
    test = list(CSDataLoader(VOCDataTestSet(str(tmp_path), str(tmp_path / "train.txt"), crop_size=(80, 90), mean=mean)))
    for i, (images, names, sizes) in enumerate(test):
        assert names == ["n%d" % i] and tuple(int(v) for v in sizes[0]) == (75, 100, 3) and images.is_cuda
        assert np.array_equal(images[0].cpu().numpy(), vp.voc_test_getitem(raws[i][0], (80, 90), mean))


# ------------------------------------------------------------------------------------------------ losses at 21 classes
@pytest.mark.parametrize("hw,HW", [((41, 41), (321, 321)), ((65, 65), (512, 512))])
def test_pixelwise_and_dsn_ce_21_classes_float64(hw, HW):
    from oracle import port
    from structure_knowledge_distillation_b200.utils.criterion import CriterionDSN, CriterionPixelWise
    g = torch.Generator().manual_seed(hw[0])
    S = [torch.randn(2, C21, *hw, generator=g) * 2 for _ in range(2)]
    T = torch.randn(2, C21, *hw, generator=g) * 2
    labels = torch.randint(0, C21, (2, *HW), generator=g)
    labels[torch.rand(2, *HW, generator=g) < 0.05] = 255
    Sd = [s.double().requires_grad_(True) for s in S]
    pi_ref = port.pixelwise_loss(Sd[0], T.double()); ce_ref = port.dsn_ce_loss(Sd, labels)
    gpi = torch.autograd.grad(pi_ref, Sd[0])[0]
    gce = torch.autograd.grad(ce_ref, Sd)
    Sg = [s.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True) for s in S]
    Tg = T.cuda().contiguous(memory_format=torch.channels_last)
    pi = CriterionPixelWise()([Sg[0]], [Tg]); pi.backward()
    gpi_mine = Sg[0].grad.clone(); Sg[0].grad = None
    ce = CriterionDSN()(Sg, labels.cuda()); ce.backward()
    rep = dict(pi=abs(float(pi) - float(pi_ref)) / float(pi_ref), ce=abs(float(ce) - float(ce_ref)) / float(ce_ref),
               d_pi=_rel(gpi_mine, gpi), d_ce0=_rel(Sg[0].grad, gce[0]), d_ce1=_rel(Sg[1].grad, gce[1]))
    print("\nPARITY losses C=21", hw, {k: "%.2e" % v for k, v in rep.items()})
    assert rep["pi"] < 1e-5 and rep["ce"] < 1e-5 and max(rep["d_pi"], rep["d_ce0"], rep["d_ce1"]) < 1e-4, rep


def test_ohem_dsn_21_classes_matches_restatement():
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN
    from tools import ohem_oracle as O
    g = torch.Generator().manual_seed(21)
    preds = [torch.randn(2, C21, 41, 41, generator=g) * 3 for _ in range(2)]
    labels = torch.randint(0, C21, (2, 321, 321), generator=g)
    labels[torch.rand(2, 321, 321, generator=g) < 0.05] = 255
    ref_in = [p.clone().requires_grad_(True) for p in preds]
    ref, thr, kept = O.ohem_dsn_loss(ref_in, labels, thresh=0.7, min_kept=20000)
    ref.backward()
    xs = [p.cuda().requires_grad_(True) for p in preds]
    crit = CriterionOhemDSN(255, 0.7, 20000)
    loss = crit(xs, labels.cuda()); loss.backward()
    rep = dict(loss=abs(float(loss) - float(ref)) / float(ref), thr=abs(float(crit.last_threshold) - thr) / thr,
               kept=abs(float(crit.last_kept) - kept) / kept, d0=_rel(xs[0].grad, ref_in[0].grad), d1=_rel(xs[1].grad, ref_in[1].grad))
    print("\nPARITY ohem C=21", {k: "%.2e" % v for k, v in rep.items()})
    assert 0 < kept < int((labels != 255).sum())
    assert rep["loss"] < 1e-4 and rep["thr"] < 1e-6 and rep["kept"] < 1e-4 and rep["d0"] < 2e-4 and rep["d1"] < 2e-4, rep


# ------------------------------------------------------------------------------------------------ the 21-class step
def _netmodel(student, batch, h, w, cfg, graph=False, **extra):
    from oracle import cases, espnet_full_port, espnet_port, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    teacher, s_port, D = cases.build_models(seed=0, with_D=True, classes=C21)
    if student == "espnet_c":
        s_port = espnet_port.build_student(7, classes=C21)
    elif student == "espnet":
        s_port = espnet_full_port.build_student(7, classes=C21)
    if not cfg.ho:
        torch.manual_seed(0)
    args = make_args(classes_num=C21, batch_size=batch, pi=cfg.pi, pa=cfg.pa, ho=cfg.ho, adv_loss_type=cfg.adv_type,
                     pool_scale=cfg.pool_scale, student=student, cuda_graph=graph, **extra)
    m = NetModel(args)
    m.student.load_state_dict(s_port.state_dict()); m.teacher.load_state_dict(teacher.state_dict()); m.D_model.load_state_dict(D.state_dict())
    images, labels = port.synthetic_batch(batch, h, w, seed=1, classes=C21)
    masks = cases.dropout_masks(s_port, batch, seed=2) if student == "resnet18" else []
    for drop, mk in zip(m.student.dropouts(), masks):
        drop.injected = mk
    if cfg.ho and cfg.adv_type == "wgan-gp":
        m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    m.set_input((images, labels, None, None))
    return m, dict(teacher=teacher, student=s_port, D=D, images=images, labels=labels, masks=masks)


def _precise_student(m):
    """Every ResNet18 student convolution forward in 3xTF32 (the default runs only the stem, layer1 and layer2 so).  At batch 1-2
    train-mode BN amplifies TF32 operand rounding in a random-init student (DESIGN.md "TF32 and parity") to a 0.36 rel-L2 of the sampled
    gradient elements at 321 x 321, which would hide a misrouted class channel; in 3xTF32 that deviation is below 1e-2."""
    from structure_knowledge_distillation_b200.networks.pspnet_combine import Conv2d
    for mod in m.student.modules():
        if isinstance(mod, Conv2d):
            mod.precise = True


def _grad_report(m, grads):
    worst, wn, sm, sg = 0.0, None, [], []
    for pname, p in m.student.named_parameters():
        gd = grads.get(pname)
        if gd is None or gd["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        e = abs(float(mine.norm()) - gd["norm"]) / gd["norm"]
        if e > worst:
            worst, wn = e, pname
        sm.append(mine[gd["idx"].to(mine.device)].cpu() / gd["norm"]); sg.append(gd["samples"].double().cpu() / gd["norm"])
    sm, sg = torch.cat(sm), torch.cat(sg)
    return (worst, wn), float((sm - sg).norm() / sg.norm()), float((sm * sg).sum() / (sm.norm() * sg.norm()))


@pytest.mark.parametrize("name", ["voc_pi_pa_ho_wgangp_512", "voc_pi_pa_321_b2"])
def test_resnet18_21_class_step_matches_reference_golden(name):
    from oracle import port
    from oracle.make_golden_steps_voc import VOC_STEP_CASES
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "steps_voc.pt"), weights_only=False)[name]
    spec = VOC_STEP_CASES[name]
    cfg = port.StepConfig(**spec["cfg"])
    m, _ = _netmodel("resnet18", spec["batch"], spec["h"], spec["w"], cfg)
    _precise_student(m)
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    assert m.preds_S[0].shape[1] == C21
    rep = dict(ce=m.mc_G_loss, G=m.G_loss, pi=m.pi_G_loss, pa=m.pa_G_loss)
    rep = {k: abs(float(v) - gold[k]) / abs(gold[k]) for k, v in rep.items()}
    rep["logits_S"] = _rel(m.preds_S[0][:, :, ::8, ::8], gold["logits_S"]); rep["logits_T"] = _rel(m.preds_T[0][:, :, ::8, ::8], gold["logits_T"])
    rep["worst_student_grad_norm_rel"], rep["student_grad_samples_rel_l2"], rep["student_grad_samples_cosine"] = \
        _grad_report(m, gold["student_grads"])
    if cfg.ho:
        m.G_solver.step(); m.discriminator_backward()
        rep["D"] = abs(float(m.D_loss) - gold["D"]) / abs(gold["D"])
    print("\nPARITY voc step", name, rep)
    for k in ("ce", "pi", "G", "D"):
        if k in rep:
            assert rep[k] < 1e-3, (k, rep[k])
    assert rep["pa"] < 1e-3
    assert rep["logits_T"] < 2e-3 and rep["logits_S"] < 2e-3
    # 3xTF32 student forward: measured 6.3e-3 / 2.1e-2 / 0.99978 at worst (batch 1 at 512 x 512)
    assert rep["worst_student_grad_norm_rel"][0] < 2e-2 and rep["student_grad_samples_rel_l2"] < 5e-2, rep
    assert rep["student_grad_samples_cosine"] > 0.999, rep


def _d_phase_vs_port(m, cfg, d_state, d_in_S, d_in_T):
    """The discriminator phase that just ran in `m` against oracle/port.py in float64 on the same logits and D state, with the
    size-aware head of the package's discriminator: -> (loss rel. error, worst D gradient rel-L2)."""
    from oracle import espnet_port, port
    Dq = port.Discriminator(1, C21, 64)
    Dq.load_state_dict({k: v.cpu() for k, v in d_state.items()})
    Dq = espnet_port.size_aware_D(Dq, tuple(d_in_S.shape[2:])).cuda().double().train()
    ls, lt = d_in_S.detach().double().contiguous(), d_in_T.detach().double().contiguous()
    dT, dS = Dq(lt), Dq(ls)
    dl = cfg.lambda_d * port.adv_loss_d(dS, dT, cfg.adv_type)
    if cfg.adv_type == "wgan-gp":
        dl = dl + cfg.lambda_d * port.gradient_penalty(Dq, ls, lt, m.criterion_AdditionalGP.alpha.double(), cfg.lambda_gp)
    dl.backward()
    refs = dict(Dq.named_parameters())
    if hasattr(Dq, "last_conv"):
        refs["last.0.weight"], refs["last.0.bias"] = Dq.last_conv.weight, Dq.last_conv.bias
    top = max(float(q.grad.norm()) for q in refs.values() if q.grad is not None)
    worst = max(float((p.grad.double() - refs[n].grad).norm() / max(float(refs[n].grad.norm()), 1e-3 * top))
                for n, p in m.D_model.named_parameters() if n in refs and refs[n].grad is not None and p.grad is not None)
    return abs(float(m.D_loss) - float(dl)) / abs(float(dl)), worst


# (student, batch, H, W): ESPNet students at sizes their strides divide; ResNet18 at VOCDataSet's default 321 x 321 crop
PORT_CASES = [("resnet18", 2, 321, 321), ("espnet_c", 2, 320, 320), ("espnet", 2, 320, 320)]


@pytest.mark.parametrize("student,batch,h,w", PORT_CASES)
@pytest.mark.parametrize("adv", ["wgan-gp", "hinge"])
def test_21_class_step_matches_float64_port(student, batch, h, w, adv):
    """Pi + Pa + Ho at 21 classes through NetModel against the students' ports in float64 on the same weights and inputs: every
    G loss within 1e-3 relative, the discriminator phase on identical logits within 1e-4, student gradient norms."""
    from oracle import cases, espnet_full_port, espnet_port, port
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type=adv)
    m, ref = _netmodel(student, batch, h, w, cfg)
    _precise_student(m)                                                # (the ESPNets run 3xTF32 throughout already)
    m.forward(); m.G_solver.zero_grad(); m.student_backward()
    assert m.preds_S[0].shape[1] == C21 and m.preds_T[0].shape[1] == C21
    T, S = ref["teacher"].cuda().double(), ref["student"].cuda().double()
    for drop, mk in zip(S.dropouts() if student == "resnet18" else [], ref["masks"]):
        drop.injected = mk.cuda().double()
    D = ref["D"]
    alpha = m.criterion_AdditionalGP.alpha.double() if adv == "wgan-gp" else None
    images, labels = ref["images"].cuda().double(), ref["labels"].cuda()
    grid = tuple(m._d_inputs()[0].shape[2:])
    D = espnet_port.size_aware_D(D, grid).cuda().double()
    step = {"resnet18": port.distill_step, "espnet_c": espnet_port.distill_step, "espnet": espnet_full_port.distill_step}[student]
    out = step(T, S, D, images, labels, cfg, gp_alpha=alpha)
    rep = {k: abs(float(v) - out[k]) / abs(out[k]) for k, v in dict(ce=m.mc_G_loss, pi=m.pi_G_loss, pa=m.pa_G_loss, G=m.G_loss).items()}
    rep["logits_S"] = _rel(m.preds_S[0], out["preds_S"][0])
    grads = cases.grad_digest(S.named_parameters())
    rep["worst_student_grad_norm_rel"], rep["student_grad_samples_rel_l2"], rep["student_grad_samples_cosine"] = _grad_report(m, grads)
    m.G_solver.step()
    d_state = {k: v.detach().clone() for k, v in m.D_model.state_dict().items()}
    with torch.no_grad():
        d_in = m._d_inputs()
    m.discriminator_backward()
    rep["D_same_inputs"], rep["worst_D_grad_same_inputs"] = _d_phase_vs_port(m, cfg, d_state, *d_in)
    print("\nPARITY voc step vs port", student, adv, rep)
    for k in ("ce", "pi", "pa", "G"):
        assert rep[k] < 1e-3, (k, rep[k])
    assert rep["D_same_inputs"] < 1e-4 and rep["worst_D_grad_same_inputs"] < 3e-3, rep
    # measured at worst: 6.1e-3 (gradient norm), 7.9e-3 (sampled elements), cosine 0.99997 -- the full ESPNet
    assert rep["worst_student_grad_norm_rel"][0] < 2e-2 and rep["student_grad_samples_rel_l2"] < 2e-2, rep
    assert rep["student_grad_samples_cosine"] > 0.999, rep


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + [p.detach().clone() for p in m.student.parameters()] + \
        [b.detach().clone() for b in m.student.buffers()] + [p.detach().clone() for p in m.D_model.parameters()]


def _same(a, b):
    return all((x == y) if isinstance(x, float) else torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("student", ["resnet18", "espnet_c", "espnet"])
def test_21_class_cuda_graph_replays_equal_eager_steps(student):
    from oracle import port
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    m, _ = _netmodel(student, 2, 320, 320, cfg)
    eager = []
    for _ in range(2):
        m.optimize_parameters(); torch.cuda.synchronize(); eager.append(_dump(m))
    del m
    m, _ = _netmodel(student, 2, 320, 320, cfg)
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
        assert _same(_dump(m), want)


@pytest.mark.parametrize("student", ["resnet18", "espnet_c", "espnet"])
def test_21_class_ohem_step(student):
    from oracle import port
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN
    from tools import ohem_oracle as O
    cfg = port.StepConfig(pi=True, pa=True, ho=False)
    m, _ = _netmodel(student, 2, 320, 320, cfg, ohem=True, ohem_thres=0.05, ohem_keep=20000)
    assert isinstance(m.criterion, CriterionOhemDSN)
    m.optimize_parameters(); torch.cuda.synchronize()
    assert float(m.G_loss) == float(m.G_loss) and 0 < float(m.criterion.last_kept) < float((m.labels != 255).sum())
    preds = [None if p is None else p.detach().float().cpu().contiguous() for p in m.preds_S[:2]]
    if preds[1] is None:
        if preds[0].shape[2:] == m.labels.shape[1:]:
            want = O.ohem_ce_loss(preds[0], m.labels.cpu(), 255, 0.05, 20000, 8)
        else:
            up = F.interpolate(preds[0], size=tuple(m.labels.shape[1:]), mode="bilinear", align_corners=True)
            want = O.ohem_ce_loss(up, m.labels.cpu(), 255, 0.05, 20000, 8)
    else:
        want = O.ohem_dsn_loss(preds, m.labels.cpu(), 255, 0.05, 20000)
    print("\nPARITY voc ohem", student, float(m.mc_G_loss), float(want[0]), float(m.criterion.last_kept), want[2])
    assert abs(float(m.mc_G_loss) - float(want[0])) <= 1e-4 * abs(float(want[0]))
    assert abs(float(m.criterion.last_kept) - want[2]) <= 1e-4 * want[2]


# ------------------------------------------------------------------------------------------------ evaluation
def _oracle_scores_sliding(ref, image, tile):
    """networks/evaluate.py's predict_sliding over a float64 oracle network: (H, W, 21) scores of a (1, 3, H, W) image."""
    import math
    _, _, H, W = image.shape
    full = torch.zeros(1, C21, H, W, dtype=torch.float64, device="cuda")
    img = image.cuda().double()
    stride = math.ceil(tile[0] * (1 - 1 / 3))
    rows, cols = int(math.ceil((H - tile[0]) / stride) + 1), int(math.ceil((W - tile[1]) / stride) + 1)
    for r in range(rows):
        for c in range(cols):
            x1, y1 = int(c * stride), int(r * stride)
            x2, y2 = min(x1 + tile[1], W), min(y1 + tile[0], H)
            x1, y1 = max(int(x2 - tile[1]), 0), max(int(y2 - tile[0]), 0)
            t = img[:, :, y1:y2, x1:x2]
            pad = torch.zeros(1, 3, tile[0], tile[1], dtype=torch.float64, device="cuda")
            pad[:, :, :t.shape[2], :t.shape[3]] = t
            with torch.no_grad():
                up = F.interpolate(ref(pad)[0], size=tile, mode="bilinear", align_corners=True)
            full[..., y1:y2, x1:x2] += up[..., :t.shape[2], :t.shape[3]]
    return full[0].permute(1, 2, 0)


def _gold_eval():
    return torch.load(gzip.open(os.path.join(ROOT, "tests", "golden", "eval_voc.pt.gz")), weights_only=False)


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_evaluate_main_on_a_voc_loader_matches_the_reference(no_tf32, tmp_path):
    """The reference's sliding-window evaluate_main at 21 classes over its VOCDataSet (tests/golden/eval_voc.pt.gz, from
    oracle/make_golden_eval_voc.py with the fixed-weight ToyNet(21)) against evaluate_main through CSDataLoader(VOCDataSet) on the
    same files and seed: the PNGs equal the reference's arg-max except at its pixels whose top-2 margin is below 1e-4 (a handful per
    image), and the IU array and mean IU equal the reference's."""
    from PIL import Image
    from oracle.make_golden_eval import ToyNet
    from structure_knowledge_distillation_b200.dataset import CSDataLoader, VOCDataSet
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    gold = _gold_eval()
    root = tmp_path / "voc"
    (root / "JPEGImages").mkdir(parents=True); (root / "SegmentationClassAug").mkdir()
    for name, (jpg, png) in gold["files"].items():
        (root / "JPEGImages" / (name + ".jpg")).write_bytes(jpg)
        (root / "SegmentationClassAug" / (name + ".png")).write_bytes(png)
    (root / "val.txt").write_text("".join(name + "\n" for name, _, _ in gold["images"]))
    ds = VOCDataSet(str(root), str(root / "val.txt"), crop_size=gold["crop"], mean=gold["mean"], scale=False, mirror=False)
    random.seed(gold["seed"]); np.random.seed(gold["seed"])
    miou, iu = evaluate_main(ToyNet(C21).cuda().eval(), CSDataLoader(ds, batch_size=1), "0", "%d,%d" % gold["crop"], C21, whole=False,
                             png_dir=str(tmp_path / "png"))
    differing = 0
    for name, r in gold["pngs"].items():
        im = Image.open(tmp_path / "png" / (name + ".png"))
        assert im.mode == r["mode"] == "P" and list(im.getpalette()) == r["palette"]
        got, want = np.array(im), r["pixels"].numpy()
        assert got.shape == want.shape == tuple(gold["crop"])
        diff = np.flatnonzero(got.reshape(-1) != want.reshape(-1))
        assert np.isin(diff, r["near_ties"].numpy()).all(), (name, diff[:20])
        assert len(r["near_ties"]) < 100, len(r["near_ties"])                 # the exclusion stays a handful of pixels
        differing += len(diff)
    print("\nPARITY voc evaluate_main vs reference: mean IU %.6f (reference %.6f), pixels differing %d" % (miou, gold["mean_IU"], differing))
    assert len(iu) == C21 and int((gold["IU"] > 0).sum()) >= 8
    tol = 1e-12 if differing == 0 else 1e-3
    assert np.abs(iu - gold["IU"].numpy()).max() <= tol and abs(miou - gold["mean_IU"]) <= tol


@pytest.mark.parametrize("student", ["resnet18", "espnet_c", "espnet"])
def test_evaluate_main_with_each_student_on_a_voc_loader(student, tmp_path):
    """The three students through evaluate_main(model, loader, '0', '512,512', 21, whole=False) over `VOCDataSet(..., crop_size=(512,
    512), scale=False, mirror=False)`, against their float64 ports: the predictions equal the port's arg-max except where its top-2
    margin is below 1e-4 (the ESPNets, 3xTF32 throughout) or below 2e-3 of the top score (ResNet18, whose eval-mode layer3 / layer4
    run on TF32 operands: logits within ~5e-4 relative of float64), and such pixels stay below 0.5 % of the image.  The IU array
    is the one the saved predictions and the labels give, and PNGs hold the whole 512 x 512 arg-max."""
    cv2 = pytest.importorskip("cv2")
    from PIL import Image
    from oracle import cases, espnet_full_port, espnet_port
    from structure_knowledge_distillation_b200.dataset import CSDataLoader, VOCDataSet
    from structure_knowledge_distillation_b200.networks import evaluate as E
    from structure_knowledge_distillation_b200.networks.espnet import ESPNet, ESPNet_C
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Res_pspnet
    if student == "resnet18":
        _, ref, _ = cases.build_models(seed=0, with_D=False, classes=C21)
        m = Res_pspnet(BasicBlock, [2, 2, 2, 2], num_classes=C21)
    else:
        ref = (espnet_port if student == "espnet_c" else espnet_full_port).build_student(7, classes=C21)
        m = (ESPNet_C if student == "espnet_c" else ESPNet)(C21)
    m.load_state_dict(ref.state_dict())
    m, ref = m.cuda().eval(), ref.cuda().double().eval()
    (tmp_path / "JPEGImages").mkdir(); (tmp_path / "SegmentationClassAug").mkdir()
    rng = np.random.default_rng(11)
    sizes = [(500, 375), (375, 500)]
    with open(tmp_path / "val.txt", "w") as f:
        for i, (h, w) in enumerate(sizes):
            cv2.imwrite(str(tmp_path / "JPEGImages" / ("v%d.jpg" % i)), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
            lab = rng.integers(0, C21, (h, w), dtype=np.uint8); lab[:, :7] = 255
            cv2.imwrite(str(tmp_path / "SegmentationClassAug" / ("v%d.png" % i)), lab)
            f.write("v%d\n" % i)
    ds = VOCDataSet(str(tmp_path), str(tmp_path / "val.txt"), crop_size=(512, 512), scale=False, mirror=False)
    loader = CSDataLoader(ds, batch_size=1)
    miou, ious = E.evaluate_main(m, loader, "0", "512,512", C21, whole=False, save_dir=str(tmp_path / "pt"), png_dir=str(tmp_path / "png"))
    conf = np.zeros((C21, C21))
    for i, (images, labels, size, name) in enumerate(CSDataLoader(ds, batch_size=1)):
        pred = torch.load(tmp_path / "pt" / ("v%d.pt" % i)).long()
        h, w = sizes[i]
        assert tuple(pred.shape) == (h, w)
        full = _oracle_scores_sliding(ref, images.cpu(), (512, 512)).cpu()[:h, :w]
        top2 = full.topk(2, dim=2).values
        tol = 2e-3 * float(top2[..., 0].abs().max()) if student == "resnet18" else 1e-4
        near = (top2[..., 0] - top2[..., 1]) < tol
        differ = pred != full.argmax(2)
        print("\nPARITY voc evaluate_main", student, name, "pixels differing:", int(differ.sum()), "near ties:", int(near.sum()))
        assert not bool((differ & ~near).any()), int((differ & ~near).sum())
        assert int(differ.sum()) < 0.005 * h * w
        png = np.array(Image.open(tmp_path / "png" / ("v%d.png" % i)))
        assert png.shape == (512, 512) and png.max() < C21 and np.array_equal(png[:h, :w], pred.numpy().astype(np.uint8))
        gt = labels[0, :h, :w].cpu().numpy()
        keep = gt != 255
        conf += np.bincount(gt[keep] * C21 + pred.numpy()[keep], minlength=C21 * C21).reshape(C21, C21)
    tp = np.diag(conf)
    want = tp / np.maximum(1.0, conf.sum(1) + conf.sum(0) - tp)
    assert len(ious) == C21 and np.array_equal(ious, want) and miou == want.mean()
    with pytest.raises(ValueError):
        E.evaluate_main(m, loader, "0", "512,512", C21, whole=False, type="test", png_dir=str(tmp_path / "png2"))


# ------------------------------------------------------------------------------------------------ two ranks
def _ddp_worker(rank, world, port_no, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port_no), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port as oport
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        res = []
        for student in ("resnet18", "espnet_c", "espnet"):
            torch.manual_seed(100 + rank)
            m = NetModel(make_args(classes_num=C21, batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world,
                                   student=student))
            p0 = m.G_solver.flat_p.clone()
            images, labels = oport.synthetic_batch(1, 320, 320, seed=7 + rank, classes=C21)
            m.set_input((images, labels, None, None))
            m.G_solver._buckets = None
            m._student_phase()
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
            assert err < 1e-6 and err2 < 1e-5, (student, err, err2)
            res.append((student, err, err2))
        if rank == 0:
            out.put(("ok", res))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_21_class_step():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29631, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nPARITY voc two ranks", res)
    assert res[0] == "ok", res
