"""Writes tests/golden/espnet_full.pt.gz: the full ESPNet (oracle/espnet_full_port.py, plain torch on the CPU in fp32) alone and as the
student of the distillation step.  `python -m oracle.make_golden_espnet_full` (a few minutes of CPU: the 360x480 steps run the
PSPNet-101 teacher).

Cases, in the layout of make_golden_espnet.py (seeded; weights are never stored -- espnet_full_port.build_student and
cases.build_models re-create them):
  * net_96x128_b2 / net_360x480_b2: train-mode forward of the full ESPNet and the backward of a seeded linear functional of its
    full-resolution logits and feat; net_96x128_b2_eval: the same in eval mode (running statistics);
  * step_pi_pa_360x480_b2 / step_pi_pa_ho_360x480_b2: the distillation step (Pi+Pa, Pi+Pa+Ho wgan-gp) under the full-resolution
    decisions of espnet_full_port (teacher logits up to 360x480, feat at 45x60, the discriminator on the teacher's 46x61 grid).
Large tensors are kept as fixed samples (cases.sample_large), gradients as cases.grad_digest fingerprints.
"""
import gzip
import io
import os

import torch

from . import cases, espnet_full_port, espnet_port, port
from .make_golden_espnet import probe

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "espnet_full.pt.gz")

NET_CASES = {
    # name: (batch, H, W, train)
    "net_96x128_b2": (2, 96, 128, True),
    "net_96x128_b2_eval": (2, 96, 128, False),
    "net_360x480_b2": (2, 360, 480, True),
}
STEP_CASES = {
    "step_pi_pa_360x480_b2": dict(batch=2, h=360, w=480, cfg=dict(pi=True, pa=True, ho=False, pool_scale=0.5)),
    "step_pi_pa_ho_360x480_b2": dict(batch=2, h=360, w=480, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
}
STUDENT_SEED = 7


def net_case(batch, h, w, train):
    m = espnet_full_port.build_student(STUDENT_SEED)
    m.train(train)
    images, _ = port.synthetic_batch(batch, h, w, seed=11)
    out = m(images)
    loss = (out[0] * probe(out[0].shape, 12)).sum() + (out[2] * probe(out[2].shape, 13)).sum()
    loss.backward()
    bn = {k: v.clone() for k, v in m.state_dict().items() if k.endswith(("running_mean", "running_var"))}
    return dict(logits=cases.sample_large(out[0].detach()), feat=cases.sample_large(out[2].detach()),
                b1=cases.sample_large(out[6].detach()), loss=float(loss), grads=cases.grad_digest(m.named_parameters()),
                running=bn)


def step_case(spec):
    cfg = port.StepConfig(**spec["cfg"])
    teacher, _, D = cases.build_models(seed=0, with_D=True)
    student = espnet_full_port.build_student(STUDENT_SEED)
    images, labels = port.synthetic_batch(spec["batch"], spec["h"], spec["w"], seed=1)
    alpha = torch.rand(spec["batch"], 1, 1, 1, generator=cases.seeded(3))
    D = espnet_port.size_aware_D(D, espnet_full_port.teacher_grid(spec["h"], spec["w"]))
    out = espnet_full_port.distill_step(teacher, student, D, images, labels, cfg, gp_alpha=alpha)
    res = {k: v for k, v in out.items() if not k.startswith("preds")}
    res["logits_S"] = out["preds_S"][0].detach()[:, :, ::16, ::16].clone()
    res["logits_T"] = out["preds_T"][0].detach()[:, :, ::16, ::16].clone()
    res["student_grads"] = cases.grad_digest(student.named_parameters())
    return res


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gold = {}
    for name, (b, h, w, train) in NET_CASES.items():
        gold[name] = net_case(b, h, w, train)
        print(name, "loss", gold[name]["loss"], flush=True)
    for name, spec in STEP_CASES.items():
        gold[name] = step_case(spec)
        print(name, {k: v for k, v in gold[name].items() if isinstance(v, float)}, flush=True)
    buf = io.BytesIO()
    torch.save(gold, buf)
    with gzip.open(GOLDEN, "wb") as f:
        f.write(buf.getvalue())
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")


def load():
    with gzip.open(GOLDEN, "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


if __name__ == "__main__":
    main()
