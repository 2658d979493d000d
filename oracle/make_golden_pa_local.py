"""Generator of tests/golden/pa_local.pt.gz: distillation steps with the local pair-wise term (oracle/pa_local_port.py) on the CPU, from
the seeded models of oracle/cases.py (the ResNet18 student) and of the students' ports (MobileNetV2, ESPNet-C) with pinned dropout masks
and WGAN-GP alpha, as make_golden_feature_kd.py pins them:

    python -m oracle.make_golden_pa_local

For every student one case puts a local term on the PSP features (scalar lambda_pa, one node per pixel) and one mixes a local x1 level
with a fully connected one (list lambda_pa).  Each case keeps the losses (one Pa term per level in list mode), sampled student logits,
gradient digests and the same samples of every parameter's update by one SGD step (lr_g, momentum, weight decay of make_args).
TEST INFRASTRUCTURE ONLY.
"""
import gzip
import io
import os
import sys
import time

import torch

from oracle import cases, espnet_port, mobilenet_port, pa_local_port, port
from oracle.make_golden_feature_kd import sgd_update

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "pa_local.pt.gz")

GOLDEN_CASES = {
    # Pi + Pa + Ho (wgan-gp), Pa local 9x9 on the 65x65 PSP features at one node per pixel
    "r18_psp_local9_pi_pa_ho_512_b1": dict(kind="resnet18", batch=1, h=512, w=512, window=9, dilation=1,
                                           cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp", pool_scale=1.0 / 65)),
    # x1 (25x33) local 9x9 at dilation 2, one node per pixel, beside the fully connected PSP term at scale 0.5
    "r18_x1_local9d2_psp_global_96x128_b2": dict(kind="resnet18", batch=2, h=96, w=128, window=[9, None, None, None, None],
                                                 dilation=[2, 1, 1, 1, 1],
                                                 cfg=dict(pi=True, pa=True, ho=False, lambda_pa=[0.5, 0.0, 0.0, 0.0, 0.5],
                                                          pool_scale=[1.0 / 25, 0.5, 0.5, 0.5, 0.5])),
    # MobileNetV2's 45x60 PSP features, local 5x5 at one node per pixel
    "mobilenetv2_psp_local5_360x480_b1": dict(kind="mobilenetv2", batch=1, h=360, w=480, window=5, dilation=1,
                                              cfg=dict(pi=True, pa=True, ho=False, pool_scale=1.0 / 45)),
    # MobileNetV2: x1 (90x120) pooled 9x12 onto 10x10 nodes, local 3x3 at dilation 4, beside a fully connected x4
    "mobilenetv2_x1_local3d4_x4_global_360x480_b1": dict(kind="mobilenetv2", batch=1, h=360, w=480, window=[3, None, None, None],
                                                         dilation=[4, 1, 1, 1],
                                                         cfg=dict(pi=True, pa=True, ho=False, lambda_pa=[0.5, 0.0, 0.0, 0.5],
                                                                  pool_scale=[0.1, 0.5, 0.5, 0.5])),
    # ESPNet-C's 45x60 PSP-level features, local 15x15 at one node per pixel (1/45)
    "espnet_c_psp_local15_360x480_b1": dict(kind="espnet_c", batch=1, h=360, w=480, window=15, dilation=1,
                                            cfg=dict(pi=True, pa=True, ho=False, pool_scale=1.0 / 45)),
    # ESPNet-C: x1 (its 180x240 b1) pooled 9x12 onto 20x20 nodes, local 7x7 at dilation 2, beside a fully connected PSP level
    "espnet_c_x1_local7d2_psp_global_360x480_b1": dict(kind="espnet_c", batch=1, h=360, w=480, window=[7, None, None, None, None],
                                                       dilation=[2, 1, 1, 1, 1],
                                                       cfg=dict(pi=True, pa=True, ho=False, lambda_pa=[0.5, 0.0, 0.0, 0.0, 0.5],
                                                                pool_scale=[0.05, 0.5, 0.5, 0.5, 0.5])),
}


def case_inputs(spec):
    """(teacher, student, D, images, labels, dropout masks, gp alpha) of a case."""
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    if spec["kind"] == "espnet_c":
        student = espnet_port.build_student(7)
    elif spec["kind"] == "mobilenetv2":
        student = mobilenet_port.build_student(7)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    masks = cases.dropout_masks(student, spec["batch"], seed=2) if spec["kind"] != "espnet_c" else []
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    return teacher, student, D, images, labels, masks, alpha


def port_step(spec):
    """The case on the CPU in fp32 -> the record the golden keeps."""
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D, images, labels, masks, alpha = case_inputs(spec)
    for drop, m in zip(student.dropouts() if masks else [], masks):
        drop.injected = m
    out = pa_local_port.distill_step(spec["kind"], teacher, student, D if cfg.ho else None, images, labels, cfg,
                                     window=spec["window"], dilation=spec["dilation"], gp_alpha=alpha)
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
        print("pa_local", name, {k: res[name][k] for k in ("ce", "pa", "G") if k in res[name]}, "%.1fs" % (time.time() - t0))
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
