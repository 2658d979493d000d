"""Generator of tests/golden/feature_kd.pt.gz: distillation steps with attention transfer and MIMIC (oracle/feature_kd_port.py) on the
CPU, from the seeded models of oracle/cases.py with pinned dropout masks and WGAN-GP alpha, as make_golden_seg.py and
tools/pa_levels_oracle.py pin them:

    python -m oracle.make_golden_feature_kd

Each case keeps the losses (one AT / MIMIC term per level in list mode), sampled student logits, gradient digests of the student and
of the MIMIC adapters, and the same samples of every parameter's update by one SGD step (lr_g, momentum, weight decay of make_args).
TEST INFRASTRUCTURE ONLY.
"""
import gzip
import io
import os
import sys
import time

import torch

from oracle import cases, espnet_port, feature_kd_port, port

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "feature_kd.pt.gz")
ADAPTER_SEED = 4

GOLDEN_CASES = {
    # every term: Pi + Pa + Ho (wgan-gp) + AT and MIMIC on the PSP features (scalar weights)
    "r18_pi_pa_ho_at_mimic_psp_512_b1": dict(kind="resnet18", batch=1, h=512, w=512, at=500.0, mimic=1.0,
                                             cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
    # AT at five levels (x2's weight 0), MIMIC at x3 alone (256 -> 1024 adapter)
    "r18_at5_mimic_x3_96x128_b2": dict(kind="resnet18", batch=2, h=96, w=128, at=[500.0, 0.0, 250.0, 500.0, 1000.0],
                                       mimic=[0.0, 0.0, 1.0], cfg=dict(pi=True, pa=False, ho=False)),
    # a resampled student: ESPNet-C's levels sit on other grids than the teacher's (b1: 19 channels at 1/2)
    "espnet_c_at5_mimic_psp_360x480_b1": dict(kind="espnet_c", batch=1, h=360, w=480, at=[500.0] * 5, mimic=1.0,
                                              cfg=dict(pi=True, pa=False, ho=False)),
}


def case_inputs(spec):
    """(teacher, student, D, adapters, images, labels, dropout masks, gp alpha) of a case."""
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    if spec["kind"] == "espnet_c":
        student = espnet_port.build_student(7)
    adapters = feature_kd_port.build_adapters(student, teacher, spec["mimic"], ADAPTER_SEED)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    masks = cases.dropout_masks(student, spec["batch"], seed=2) if spec["kind"] == "resnet18" else []
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    return teacher, student, D, adapters, images, labels, masks, alpha


def sgd_update(named_params, digest, cfg):
    """p_after - p at the digest's sample positions for the first step of torch.optim.SGD (momentum buffer = grad + wd * p)."""
    out = {}
    for name, p in named_params:
        if name in digest:
            idx = digest[name]["idx"]
            g, w = p.grad.detach().flatten().double()[idx], p.detach().flatten().double()[idx]
            out[name] = (-cfg.lr_g * (g + cfg.weight_decay * w)).float()
    return out


def port_step(spec):
    """The case on the CPU in fp32 -> the record the golden keeps."""
    cfg = port.StepConfig(**spec["cfg"])
    teacher, student, D, adapters, images, labels, masks, alpha = case_inputs(spec)
    for drop, m in zip(student.dropouts() if masks else [], masks):
        drop.injected = m
    out = feature_kd_port.distill_step(spec["kind"], teacher, student, D if cfg.ho else None, adapters, images, labels, cfg,
                                       at=spec["at"], mimic=spec["mimic"], gp_alpha=alpha)
    rec = {k: v for k, v in out.items() if not k.startswith("preds")}
    rec["logits_S"] = out["preds_S"][0].detach()[:, :, ::8, ::8].clone()
    rec["student_grads"] = cases.grad_digest(student.named_parameters())
    rec["adapter_grads"] = cases.grad_digest(adapters.named_parameters())
    rec["student_update"] = sgd_update(student.named_parameters(), rec["student_grads"], cfg)
    rec["adapter_update"] = sgd_update(adapters.named_parameters(), rec["adapter_grads"], cfg)
    if cfg.ho:
        rec["D_grads"] = cases.grad_digest(D.named_parameters())
    return rec


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    res = {}
    for name, spec in GOLDEN_CASES.items():
        t0 = time.time()
        res[name] = port_step(spec)
        print("feature_kd", name, {k: res[name][k] for k in ("ce", "at", "mimic", "G") if k in res[name]}, "%.1fs" % (time.time() - t0))
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
