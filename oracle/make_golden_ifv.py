"""Generator of tests/golden/ifv.pt.gz: distillation steps with intra-class feature variation distillation (oracle/ifv_port.py) on the
CPU, from the seeded models of oracle/cases.py with pinned dropout masks and WGAN-GP alpha, as make_golden_cwd.py pins them:

    python -m oracle.make_golden_ifv

Each case keeps the losses (out["ifv"]: the term, a list for list weights), sampled student logits, the student's gradient digest and
the same samples of its update by one SGD step (lr_g, momentum, weight decay of make_args).  TEST INFRASTRUCTURE ONLY.
"""
import gzip
import io
import os
import sys
import time

import torch

from oracle import cases, espnet_port, feature_kd_port, ifv_port, mobilenet_port, port
from oracle.make_golden_feature_kd import sgd_update

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ifv.pt.gz")

GOLDEN_CASES = {
    # every term of the paper plus IFV on the PSP features (128 student against 512 teacher channels), as IFVD trains it
    "r18_pi_pa_ho_ifv_psp_512_b1": dict(kind="resnet18", classes=19, batch=1, h=512, w=512, ifv=200.0, lambda_cwd=0.0,
                                        cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
    # IFV on all five levels (x1 .. x4 and the PSP features) beside CWD on the logits
    "r18_ifv_levels_cwd_96x128_b2": dict(kind="resnet18", classes=19, batch=2, h=96, w=128, ifv=[200.0] * 5, lambda_cwd=3.0,
                                         cfg=dict(pi=True, pa=False, ho=False)),
    # ESPNet-C: its PSP level (46x61 against the teacher's 45x60 at 360x480) on the resampled teacher, the labels taken to 46x61
    "espnet_c_ifv_psp_360x480_b1": dict(kind="espnet_c", classes=19, batch=1, h=360, w=480, ifv=200.0, lambda_cwd=0.0,
                                        cfg=dict(pi=True, pa=False, ho=False)),
    # MobileNetV2 at 21 classes (PASCAL VOC's count), synthetic labels over 0..20 and 255
    "mbv2_ifv_psp_voc21_96x128_b2": dict(kind="mobilenetv2", classes=21, batch=2, h=96, w=128, ifv=200.0, lambda_cwd=0.0,
                                         cfg=dict(pi=True, pa=False, ho=False)),
}


def case_inputs(spec):
    """(teacher, student, D, images, labels, dropout masks, gp alpha) of a case."""
    teacher, student, D = cases.build_models(seed=0, with_D=True, classes=spec["classes"])
    if spec["kind"] == "espnet_c":
        student = espnet_port.build_student(7)
    elif spec["kind"] == "mobilenetv2":
        student = mobilenet_port.build_student(7, classes=spec["classes"])
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1, classes=spec["classes"])
    masks = cases.dropout_masks(student, spec["batch"], seed=2) if spec["kind"] in ("resnet18", "mobilenetv2") else []
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    return teacher, student, D, images, labels, masks, alpha


def port_step(spec):
    """The case on the CPU in fp32 -> the record the golden keeps."""
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D, images, labels, masks, alpha = case_inputs(spec)
    for drop, m in zip(student.dropouts() if masks else [], masks):
        drop.injected = m
    out = ifv_port.distill_step(spec["kind"], teacher, student, D if cfg.ho else None, {}, {}, images, labels, cfg,
                                lambda_cwd=spec["lambda_cwd"], ifv=spec["ifv"], classes_num=spec["classes"], gp_alpha=alpha)
    rec = {k: v for k, v in out.items() if not k.startswith("preds")}
    rec["logits_S"] = out["preds_S"][0].detach()[:, :, ::8, ::8].clone()
    rec["student_grads"] = cases.grad_digest(student.named_parameters())
    rec["student_update"] = sgd_update(student.named_parameters(), rec["student_grads"], cfg)
    if cfg.ho:
        rec["D_grads"] = cases.grad_digest(D.named_parameters())
    return rec


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    res = {}
    for name, spec in GOLDEN_CASES.items():
        t0 = time.time()
        res[name] = port_step(spec)
        print("ifv", name, {k: res[name][k] for k in ("ce", "cwd", "ifv", "G") if k in res[name]}, "%.1fs" % (time.time() - t0))
    buf = io.BytesIO()
    torch.save(res, buf)
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(buf.getvalue())
    print("written", GOLDEN, "torch", torch.__version__)


def load():
    with gzip.open(GOLDEN, "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


if __name__ == "__main__":
    sys.exit(main())
