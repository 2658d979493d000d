"""Generator of tests/golden/cwd.pt.gz: distillation steps with channel-wise distillation (oracle/cwd_port.py) on the CPU, from the
seeded models of oracle/cases.py with pinned dropout masks and WGAN-GP alpha, as make_golden_feature_kd.py pins them:

    python -m oracle.make_golden_cwd

Each case keeps the losses (out["cwd"]: the logit term, or [logits, level 0, ...] with feature levels), sampled student logits,
gradient digests of the student and of both adapter families (MIMIC's and CWD's), and the same samples of every parameter's update by
one SGD step (lr_g, momentum, weight decay of make_args).  TEST INFRASTRUCTURE ONLY.
"""
import gzip
import io
import os
import sys
import time

import torch

from oracle import cases, cwd_port, espnet_full_port, espnet_port, feature_kd_port, port
from oracle.make_golden_feature_kd import ADAPTER_SEED, sgd_update

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "cwd.pt.gz")
CWD_ADAPTER_SEED = 5

GOLDEN_CASES = {
    # every term of the paper plus CWD on the logits
    "r18_pi_pa_ho_cwd_logits_512_b1": dict(kind="resnet18", batch=1, h=512, w=512, lambda_cwd=3.0, cwd_feat=None, mimic=None,
                                           cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
    # CWD on the logits and at x3, x4 and the PSP features (256 -> 1024, 512 -> 2048, 128 -> 512 adapters), MIMIC at x3 too: two
    # adapter families in the flat buffer, one level with both
    "r18_cwd_levels_mimic_x3_96x128_b2": dict(kind="resnet18", batch=2, h=96, w=128, lambda_cwd=3.0, cwd_feat=[0.0, 0.0, 1.0, 1.0, 1.0],
                                              mimic=[0.0, 0.0, 1.0], cfg=dict(pi=True, pa=False, ho=False)),
    # the full ESPNet: CWD on its input-resolution logits against the teacher's logits resized onto 360x480
    "espnet_cwd_logits_360x480_b1": dict(kind="espnet", batch=1, h=360, w=480, lambda_cwd=3.0, cwd_feat=None, mimic=None,
                                         cfg=dict(pi=True, pa=False, ho=False)),
    # ESPNet-C: its PSP-level features (46x61 against the teacher's 45x60 at 360x480) resampled, no logit term
    "espnet_c_cwd_psp_360x480_b1": dict(kind="espnet_c", batch=1, h=360, w=480, lambda_cwd=0.0, cwd_feat=2.0, mimic=None,
                                        cfg=dict(pi=True, pa=False, ho=False)),
}


def case_inputs(spec):
    """(teacher, student, D, MIMIC adapters, CWD adapters, images, labels, dropout masks, gp alpha) of a case."""
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    if spec["kind"] == "espnet_c":
        student = espnet_port.build_student(7)
    elif spec["kind"] == "espnet":
        student = espnet_full_port.build_student(7)
    mimic = feature_kd_port.build_adapters(student, teacher, spec["mimic"], ADAPTER_SEED)
    cwd = feature_kd_port.build_adapters(student, teacher, spec["cwd_feat"], CWD_ADAPTER_SEED)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    masks = cases.dropout_masks(student, spec["batch"], seed=2) if spec["kind"] == "resnet18" else []
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    return teacher, student, D, mimic, cwd, images, labels, masks, alpha


def port_step(spec):
    """The case on the CPU in fp32 -> the record the golden keeps."""
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D, mimic, cwd, images, labels, masks, alpha = case_inputs(spec)
    for drop, m in zip(student.dropouts() if masks else [], masks):
        drop.injected = m
    out = cwd_port.distill_step(spec["kind"], teacher, student, D if cfg.ho else None, mimic, cwd, images, labels, cfg,
                                mimic=spec["mimic"], lambda_cwd=spec["lambda_cwd"], cwd_feat=spec["cwd_feat"], gp_alpha=alpha)
    rec = {k: v for k, v in out.items() if not k.startswith("preds")}
    rec["logits_S"] = out["preds_S"][0].detach()[:, :, ::8, ::8].clone()
    rec["student_grads"] = cases.grad_digest(student.named_parameters())
    rec["student_update"] = sgd_update(student.named_parameters(), rec["student_grads"], cfg)
    for fam, ad in (("mimic", mimic), ("cwd", cwd)):
        rec[fam + "_adapter_grads"] = cases.grad_digest(ad.named_parameters())
        rec[fam + "_adapter_update"] = sgd_update(ad.named_parameters(), rec[fam + "_adapter_grads"], cfg)
    if cfg.ho:
        rec["D_grads"] = cases.grad_digest(D.named_parameters())
    return rec


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    res = {}
    for name, spec in GOLDEN_CASES.items():
        t0 = time.time()
        res[name] = port_step(spec)
        print("cwd", name, {k: res[name][k] for k in ("ce", "mimic", "cwd", "G") if k in res[name]}, "%.1fs" % (time.time() - t0))
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
