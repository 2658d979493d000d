"""Full distillation steps with the holistic loss at crops whose discriminator attention sees more than 128 positions, on the H100.

769x769 (the standard Cityscapes training crop: 97x97 logits, attn1 over 144 positions) and the full 1024x2048 frame (129x257
logits, attn1 over 512).  Each step runs through NetModel; its discriminator phase is checked against oracle/port.py in float64
(autograd, double backward for the penalty) fed with the step's own teacher / student logits and D state.  At 769x769 the whole
step is also checked against the UNMODIFIED reference (tests/golden/steps_769.pt, oracle/make_golden_large_crop.py), and a
CUDA-graph replay of the step equals the eager step bit for bit."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _relerr(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _netmodel(batch, h, w):
    from oracle import cases, port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp"))
    m.student.load_state_dict(student.state_dict()); m.teacher.load_state_dict(teacher.state_dict()); m.D_model.load_state_dict(D.state_dict())
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    for drop, mk in zip(m.student.dropouts(), cases.dropout_masks(student, batch, seed=2)):
        drop.injected = mk
    m.criterion_AdditionalGP.alpha = torch.rand(batch, 1, 1, 1, generator=cases.seeded(3)).cuda()
    m.set_input((images, labels, None, None))
    return m, cfg


def _d_phase_vs_port(m, cfg, d_state):
    """The discriminator phase that just ran in `m` against oracle/port.py in float64 on the same logits and D state.
    -> (loss rel. error, (worst whole-tensor grad rel-L2, name))"""
    from oracle import port
    Dq = port.Discriminator(1, 19, 64)
    Dq.load_state_dict({k: v.cpu() for k, v in d_state.items()})
    Dq = Dq.cuda().double().train()
    tf = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False; torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ls, lt = m.preds_S[0].detach().double().contiguous(), m.preds_T[0].detach().double().contiguous()
        dT, dS = Dq(lt), Dq(ls)                                                     # kd_model.py:156-157 order
        dl = cfg.lambda_d * port.adv_loss_d(dS, dT, cfg.adv_type)
        dl = dl + cfg.lambda_d * port.gradient_penalty(Dq, ls, lt, m.criterion_AdditionalGP.alpha.double(), cfg.lambda_gp)
        dl.backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf
    refs = dict(Dq.named_parameters())
    topq = max(float(q.grad.norm()) for q in refs.values() if q.grad is not None)
    wq, wqn = 0.0, None
    for pname, p in m.D_model.named_parameters():
        q = refs.get(pname)
        if q is None or q.grad is None or p.grad is None:
            continue
        e = float((p.grad.detach().double() - q.grad).norm() / max(float(q.grad.norm()), 1e-3 * topq))
        if e > wq:
            wq, wqn = e, pname
    return abs(float(m.D_loss) - float(dl)) / max(abs(float(dl)), 1e-12), (wq, wqn)


@pytest.mark.parametrize("batch,h,w,logits,n1", [(2, 769, 769, (97, 97), 144), (1, 1024, 2048, (129, 257), 512)])
def test_holistic_step_at_large_crops(batch, h, w, logits, n1):
    """Pi + Pa + Ho (wgan-gp) through NetModel; the D phase within the bounds of the 360x480 holistic step test on identical inputs."""
    m, cfg = _netmodel(batch, h, w)
    m.forward(); m.G_solver.zero_grad(); m.student_backward(); m.G_solver.step()
    assert tuple(m.preds_S[0].shape[2:]) == logits
    d_state = {k: v.detach().clone() for k, v in m.D_model.state_dict().items()}
    m.discriminator_backward()
    e_loss, worst = _d_phase_vs_port(m, cfg, d_state)
    print("\nPARITY ho_step %dx%d b%d (attn1 n = %d): D loss %.2e worst D grad rel-L2 (identical inputs) %.2e (%s) G %.4f D %.4f"
          % (h, w, batch, n1, e_loss, worst[0], worst[1], float(m.G_loss), float(m.D_loss)))
    assert e_loss < 1e-4 and worst[0] < 3e-2
    for v in (m.G_loss, m.D_loss, m.pi_G_loss, m.pa_G_loss):
        assert float(v) == float(v)                                            # finite


def test_step_at_769_matches_reference_golden():
    """NetModel at 769x769, batch 1, Pi + Pa + Ho wgan-gp, against tests/golden/steps_769.pt (the UNMODIFIED reference on the CPU,
    oracle/make_golden_large_crop.py), with the bounds of the 512x512 wgan-gp case of tests/test_step_gpu.py: losses within 1e-3
    (Pa 5e-3), logits, student gradient norms and sampled elements, and the discriminator phase against oracle/port.py on identical
    inputs plus its gradient norms against the golden."""
    from oracle import cases
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "steps_769.pt"), weights_only=False)["pi_pa_ho_wgangp_769"]
    m, cfg = _netmodel(1, 769, 769)
    m.forward()
    m.G_solver.zero_grad()
    m.student_backward()
    rep = {k: _relerr(v, gold[k]) for k, v in dict(ce=m.mc_G_loss, pi=m.pi_G_loss, pa=m.pa_G_loss, G=m.G_loss).items()}
    for key, t in (("logits_S", m.preds_S[0]), ("logits_T", m.preds_T[0])):
        mine, ref = cases.at_stored(t[:, :, ::8, ::8].float().cpu(), gold[key])
        rep[key] = float((mine - ref).norm() / ref.norm())
    rep["feat_T_norm"] = _relerr(m.preds_T[2].norm(), gold["feat_T_norm"])
    worst, samp_mine, samp_gold = (0.0, None), [], []
    for pname, p in m.student.named_parameters():
        g = gold["student_grads"].get(pname)
        if g is None or g["norm"] < 1e-6:
            continue
        mine = p.grad.detach().flatten().double()
        worst = max(worst, (abs(float(mine.norm()) - g["norm"]) / g["norm"], pname))
        samp_mine.append(mine[g["idx"].to(mine.device)].cpu() / g["norm"]); samp_gold.append(g["samples"].double() / g["norm"])
    sm, sg = torch.cat(samp_mine), torch.cat(samp_gold)
    rep["worst_student_grad_norm_rel"] = worst
    rep["student_grad_samples_rel_l2"] = float((sm - sg).norm() / sg.norm())
    rep["student_grad_samples_cosine"] = float((sm * sg).sum() / (sm.norm() * sg.norm()))
    m.G_solver.step()
    d_state = {k: v.detach().clone() for k, v in m.D_model.state_dict().items()}
    m.discriminator_backward()
    rep["D"] = _relerr(m.D_loss, gold["D"])
    rep["D_same_inputs"], rep["worst_D_grad_rel_l2_same_inputs"] = _d_phase_vs_port(m, cfg, d_state)
    top = max(g["norm"] for g in gold["D_grads"].values())
    wd = (0.0, None)
    for pname, p in m.D_model.named_parameters():
        g = gold["D_grads"].get(pname)
        if g is None or p.grad is None:
            continue
        wd = max(wd, (abs(float(p.grad.detach().double().norm()) - g["norm"]) / max(g["norm"], 1e-3 * top), pname))
    rep["worst_D_grad_norm_rel"] = wd
    print("\nPARITY step_769_vs_reference", {k: (("%.2e" % v) if isinstance(v, float) else v) for k, v in rep.items()})
    for k in ("ce", "pi", "pa", "G", "D"):
        assert rep[k] < (5e-3 if k == "pa" else 1e-3), (k, rep[k])
    assert rep["logits_T"] < 2e-3 and rep["logits_S"] < 3e-2
    assert rep["worst_student_grad_norm_rel"][0] < 0.6, rep["worst_student_grad_norm_rel"]
    assert rep["student_grad_samples_rel_l2"] < 0.35 and rep["student_grad_samples_cosine"] > 0.93
    assert rep["D_same_inputs"] < 1e-4 and rep["worst_D_grad_rel_l2_same_inputs"][0] < 3e-2
    assert rep["worst_D_grad_norm_rel"][0] < 0.3, rep["worst_D_grad_norm_rel"]


def _dump(m):
    return [float(m.G_loss), float(m.D_loss)] + [p.detach().clone() for mod in (m.student, m.D_model) for p in mod.parameters()] + \
        [b.detach().clone() for mod in (m.student, m.D_model) for b in mod.buffers()]


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


def test_cuda_graph_replay_equals_eager_step_at_769():
    """769x769 batch 2, Pi + Pa + Ho (wgan-gp): two replays of the captured step, rewound to the starting state, equal two eager steps
    from that state bit for bit (losses, every student and discriminator parameter and buffer)."""
    m, _ = _netmodel(2, 769, 769)
    eager = []
    for _ in range(2):
        m.optimize_parameters()
        torch.cuda.synchronize()
        eager.append(_dump(m))
    del m
    m, _ = _netmodel(2, 769, 769)
    snap = _state(m)
    m.enable_cuda_graphs(warmup=1)
    m.optimize_parameters(); m.optimize_parameters()                     # eager warm-up, capture
    assert m._graphs["captured"]
    _rewind(m, snap)
    for want in eager:
        m.optimize_parameters()
        torch.cuda.synchronize()
        assert _same(_dump(m), want)
