"""Cost of the MobileNetV2 student: the distillation step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs) with the ResNet18-PSP
and MobileNetV2 students, alternated within one run, and CUDA-event times of the depthwise kernels at the backbone's shapes, as GB/s
against a torch device-to-device copy of the same bytes.

    python -m tools.mobilenet_step_bench --steps 10 --warmup 4 --rounds 2

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the rates do not depend
on the values."""
import argparse
import json

import torch

from tools.espnet_step_bench import _time, card


def step_rate(student, batch, h, w, steps, warmup):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", student=student, cuda_graph=True))
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
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


# (name, C, H, W of the input at 512x1024, stride, dilation): one depthwise layer of each (stride, dilation) the backbone has
DW_LAYERS = (("f1_32ch_s1d1", 32, 256, 512, 1, 1), ("f2_96ch_s2d1", 96, 256, 512, 2, 1), ("f4_144ch_s2d1", 144, 128, 256, 2, 1),
             ("f8_384ch_s1d2", 384, 64, 128, 1, 2), ("f15_960ch_s1d4", 960, 64, 128, 1, 4))


def depthwise_rates(batch):
    """ms per call and GB/s (compulsory bytes: input read once, output written once; the weight gradient reads x and dy) of the
    forward (with the fused BatchNorm statistics), data gradient and weight gradient, beside a torch copy of the same bytes."""
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {}
    for name, c, h, w, s, d in DW_LAYERS:
        oh, ow = (h - 1) // s + 1, (w - 1) // s + 1
        x = ops.empty_nhwc(batch, c, h, w, "cuda"); x.normal_(generator=g)
        dy = ops.empty_nhwc(batch, c, oh, ow, "cuda"); dy.normal_(generator=g)
        wt = torch.randn(c, 1, 3, 3, device="cuda", generator=g)
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        nbytes = 4.0 * batch * c * (h * w + oh * ow)
        src = torch.empty(int(nbytes // 8), device="cuda"); dst = torch.empty_like(src)
        t = dict(fwd_stats=_time(lambda: ops.dwconv3x3_fwd(x, wt, s, d, True, 0.1, rm, rv), 50),
                 dgrad=_time(lambda: ops.dwconv3x3_dgrad(dy, wt, (batch, c, h, w), s, d), 50),
                 wgrad=_time(lambda: ops.dwconv3x3_wgrad(x, dy, s, d), 50),
                 copy_same_bytes=_time(lambda: dst.copy_(src), 50))
        out[name] = {k: dict(ms=round(v, 4), GBps=round(nbytes / v / 1e6, 1)) for k, v in t.items()}
        del x, dy, src, dst
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, shape="512x1024", losses="Pi+Pa+Ho wgan-gp", cuda_graph=True, resnet18=[], mobilenetv2=[])
    for _ in range(a.rounds):
        for student in ("resnet18", "mobilenetv2"):
            ips, ms = step_rate(student, a.batch, 512, 1024, a.steps, a.warmup)
            res[student].append(dict(images_per_s=round(ips, 2), ms_per_step=round(ms, 2)))
    res["depthwise"] = depthwise_rates(a.batch)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
