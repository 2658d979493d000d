"""TEST INFRASTRUCTURE -- generates tests/golden/steps_voc.pt: 21-class (PASCAL VOC) distillation steps of the UNMODIFIED reference,
on the CPU, with the ResNet18-PSP student and the PSPNet-101 teacher (the reference's `Res_pspnet` default class count), pinning
oracle/port.py at 21 classes on the spot.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_steps_voc

Cases (`VOC_STEP_CASES`): batch 1 at 512 x 512 with Pi + Pa + Ho wgan-gp (the reference discriminator needs 65 x 65 logits), and
batch 2 at 321 x 321, `VOCDataSet`'s default crop (41 x 41 logits), with Pi + Pa: the reference discriminator cannot run there, so
tests/test_voc_gpu.py checks Ho at that size against oracle/port.py's size-aware head.  Same seeds and step order as
oracle/make_golden.py's 19-class cases.
"""
import os
import time

import torch

from . import cases, port, refshim
from .make_golden import GOLDEN_DIR, _ref_step, _rel

CLASSES = 21
VOC_STEP_CASES = {
    "voc_pi_pa_ho_wgangp_512": dict(batch=1, h=512, w=512, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
    "voc_pi_pa_321_b2": dict(batch=2, h=321, w=321, cfg=dict(pi=True, pa=True, ho=False)),
}


def main():
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count())
    res = {}
    for name, spec in VOC_STEP_CASES.items():
        t0 = time.time()
        cfg = port.StepConfig(**spec["cfg"])
        teacher, student, D = cases.build_models(seed=0, with_D=cfg.ho, classes=CLASSES)
        images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1, classes=CLASSES)
        masks = cases.dropout_masks(student, spec["batch"], seed=2)
        alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
        P = ref.pspnet
        r_student = P.Res_pspnet(P.BasicBlock, [2, 2, 2, 2], num_classes=CLASSES)
        r_teacher = P.Res_pspnet(P.Bottleneck, [3, 4, 23, 3], num_classes=CLASSES)
        r_student.load_state_dict(student.state_dict(), strict=True)
        r_teacher.load_state_dict(teacher.state_dict(), strict=True)
        r_D = None
        if cfg.ho:
            r_D = ref.sagan.Discriminator(1, CLASSES, spec["batch"], 65, 64)
            r_D.load_state_dict(D.state_dict(), strict=True)
        for drop, m in zip(student.dropouts(), masks):
            drop.injected = m
        for (holder, idx), m in zip(((r_student.pspmodule.bottleneck, 2), (r_student.dsn, 2)), masks):
            cd = port.ChannelDropout(0.1); cd.injected = m
            holder[idx] = cd
        gold = _ref_step(ref, r_teacher, r_student, r_D, images, labels, cfg, alpha)
        mine = port.distill_step(teacher, student, D, images, labels, cfg, gp_alpha=alpha)
        for k in ("ce", "pi", "pa", "adv_g", "G", "D"):
            if k in gold:
                assert _rel(mine[k], gold[k]) < 2e-4, (name, k, mine[k], gold[k])
        mg = cases.grad_digest(student.named_parameters())
        worst = max(_rel(mg[k]["norm"], v["norm"]) for k, v in gold["student_grads"].items() if v["norm"] > 1e-6)
        assert worst < 5e-3, (name, worst)
        print("step", name, {k: round(v, 6) for k, v in gold.items() if isinstance(v, float)},
              "port grad-norm worst rel %.2e" % worst, "%.1fs" % (time.time() - t0))
        res[name] = gold
    out = os.path.join(GOLDEN_DIR, "steps_voc.pt")
    torch.save(res, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KB")


if __name__ == "__main__":
    main()
