"""Cost of the class-weighted task loss at the CamVid shape: the 11-class distillation step (batch 16 at 360x480, Pi+Pa+Ho wgan-gp,
CUDA graphs) of the ResNet18, ESPNet-C and ESPNet students, each with and without ENet class weights, alternated within one run;
and the DSN cross-entropy kernels alone (training forward + column phase) on each student's logits at that shape, weighted and
unweighted.

    python -m tools.camvid_step_bench --steps 20 --warmup 5 --rounds 3

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the rates do not depend
on the values."""
import argparse
import json

import torch

from tools.espnet_step_bench import _time, card

C = 11
STUDENTS = ("resnet18", "espnet_c", "espnet")
# the task-loss logits of each student at 360x480: (heads, h, w)
LOGITS = {"resnet18": (2, 45, 60), "espnet_c": (1, 45, 60), "espnet": (1, 360, 480)}


def _weights(labels):
    valid = labels[labels != 255]
    p = torch.bincount(valid, minlength=C).double() / valid.numel()
    return (1.0 / torch.log(1.02 + p)).float()


def step_rate(student, weighted, batch, steps, warmup):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    images, labels = port.synthetic_batch(batch, 360, 480, seed=1, classes=C)
    m = NetModel(make_args(classes_num=C, batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", student=student,
                           cuda_graph=True, class_weights=_weights(labels) if weighted else None))
    m.set_input((images, labels, None, None))
    for _ in range(warmup):
        m.optimize_parameters()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.optimize_parameters()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del m
    torch.cuda.empty_cache()
    return batch * 1000.0 / ms, ms


def ce_kernels_ms(student, weighted, batch):
    """ops.dsn_ce_fwd_train + ops.dsn_ce_bwd_cols on the student's NHWC logits against 360x480 labels."""
    from structure_knowledge_distillation_b200 import ops
    heads, h, w = LOGITS[student]
    g = torch.Generator(device="cuda").manual_seed(h)
    ls = [torch.randn(batch, C, h, w, device="cuda", generator=g).contiguous(memory_format=torch.channels_last) for _ in range(heads)]
    labels = torch.randint(0, C, (batch, 360, 480), device="cuda", generator=g)
    l1, w1 = (ls[1], 0.4) if heads == 2 else (None, 0.0)
    weight = _weights(labels).cuda() if weighted else None
    go = torch.ones((), device="cuda")

    def run():
        out, rows = ops.dsn_ce_fwd_train(ls[0], l1, labels, 255, 1.0, w1, weight)
        ops.dsn_ce_bwd_cols(ls[0], l1, rows, 360, 1.0, w1, go, out[1])
    return _time(run, 100)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, shape="360x480", classes=C, losses="Pi+Pa+Ho wgan-gp", cuda_graph=True, steps={})
    for _ in range(a.rounds):
        for s in STUDENTS:
            for weighted in (False, True):
                ips, ms = step_rate(s, weighted, a.batch, a.steps, a.warmup)
                key = "%s_%s" % (s, "weighted" if weighted else "unweighted")
                res["steps"].setdefault(key, []).append(dict(images_per_s=round(ips, 2), ms_per_step=round(ms, 2)))
    res["ce_fwd_train_bwd_cols_ms"] = {}
    for _ in range(3):
        for s in STUDENTS:
            for weighted in (False, True):
                key = "%s_%s" % (s, "weighted" if weighted else "unweighted")
                res["ce_fwd_train_bwd_cols_ms"].setdefault(key, []).append(round(ce_kernels_ms(s, weighted, a.batch), 4))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
