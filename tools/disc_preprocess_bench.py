"""Cost of the discriminator phase in each input mode (preprocess_GAN_mode 1 = BatchNorm2d, 2 = tanh, 3 = rescale).

The discriminator phase of a Pi + Pa + Ho wgan-gp step (D(T), D(S), adversarial loss, gradient penalty, backward, D update), eager,
batch 8 at 512x1024: for each mode the student's forward, backward and update run first, then a synchronise, then the discriminator
phase alone between two CUDA events.  The three modes are alternated within one run, `--rounds` times.

    python -m tools.disc_preprocess_bench --steps 10 --warmup 3 --rounds 2

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the times do not depend
on the values."""
import argparse
import json

import torch

from tools.espnet_step_bench import card


def d_phase_ms(mode, batch, h, w, steps, warmup):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", preprocess_GAN_mode=mode))
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    times = []
    for i in range(warmup + steps):
        m.forward(); m.G_solver.zero_grad(); m.student_backward(); m.G_solver.step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m.discriminator_backward()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(e0.elapsed_time(e1))
    del m
    torch.cuda.empty_cache()
    times.sort()
    return dict(mean=round(sum(times) / len(times), 3), median=round(times[len(times) // 2], 3), min=round(times[0], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--h", type=int, default=512)
    ap.add_argument("--w", type=int, default=1024)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, crop="%dx%d" % (a.h, a.w), losses="Pi+Pa+Ho wgan-gp", timed="discriminator phase, eager",
               d_phase_ms={"mode1_bn": [], "mode2_tanh": [], "mode3_rescale": []})
    names = {1: "mode1_bn", 2: "mode2_tanh", 3: "mode3_rescale"}
    for r in range(a.rounds):
        order = (1, 2, 3) if r % 2 == 0 else (3, 2, 1)
        for mode in order:
            res["d_phase_ms"][names[mode]].append(d_phase_ms(mode, a.batch, a.h, a.w, a.steps, a.warmup))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
