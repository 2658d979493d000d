"""Speed and memory of SegModel's training step (no teacher, no discriminator): PSPNet-ResNet101 at 512x1024 and at 769x769, and the
ResNet18-PSP baseline at 512x1024, beside NetModel's step with every distillation term off (pi = pa = ho = False), which still runs the
frozen teacher.  Images/s from CUDA events over `--steps` CUDA-graph replays after `--warmup` steps, and the peak allocation
(torch.cuda.max_memory_allocated) of each configuration from a fresh model.  With `--profile`, one eager ResNet101 step at 512x1024
under torch.profiler, its kernel time summed by kernel name (the top entries).

    python -m tools.seg_step_bench --steps 10 --warmup 4 --rounds 2 [--profile]

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the rates do not depend
on the values."""
import argparse
import json

import torch

from tools.espnet_step_bench import card

CONFIGS = (("resnet101", 512, 1024), ("resnet101", 769, 769), ("resnet18", 512, 1024))


def _model(kind, batch, graph, netmodel=False):
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    if netmodel:
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        return NetModel(make_args(batch_size=batch, pi=False, pa=False, ho=False, student=kind, cuda_graph=graph))
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    return SegModel(make_args(batch_size=batch, seg_model=kind, cuda_graph=graph))


def step_rate(kind, batch, h, w, steps, warmup, netmodel=False):
    from oracle import port
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = _model(kind, batch, True, netmodel)
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
    loss = float(m.G_loss)
    peak = torch.cuda.max_memory_allocated()
    del m
    torch.cuda.empty_cache()
    return dict(images_per_s=round(batch * 1000.0 / ms, 2), ms_per_step=round(ms, 2), peak_GB=round(peak / 1e9, 2), loss=round(loss, 4))


def profile_step(batch, h, w, top=25):
    """Kernel time of one eager ResNet101 step, summed by kernel name -> (total ms, [(name, ms, launches)])."""
    from torch.profiler import ProfilerActivity, profile
    from oracle import port
    m = _model("resnet101", batch, False)
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    for _ in range(2):
        m.optimize_parameters()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.optimize_parameters()
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            t, n = agg.get(e.name, (0.0, 0))
            agg[e.name] = (t + e.device_time_total / 1000.0, n + 1)
    total = sum(t for t, _ in agg.values())
    rows = sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]
    del m
    torch.cuda.empty_cache()
    return round(total, 2), [(k[:120], round(t, 3), n) for k, (t, n) in rows]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, cuda_graph=True, seg={}, netmodel_no_distillation={})
    for _ in range(a.rounds):
        for kind, h, w in CONFIGS:
            res["seg"].setdefault("%s_%dx%d" % (kind, h, w), []).append(step_rate(kind, a.batch, h, w, a.steps, a.warmup))
        res["netmodel_no_distillation"].setdefault("resnet18_512x1024", []).append(
            step_rate("resnet18", a.batch, 512, 1024, a.steps, a.warmup, netmodel=True))
    if a.profile:
        total, rows = profile_step(a.batch, 512, 1024)
        res["profile_resnet101_512x1024"] = dict(kernel_ms=total, top=rows)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
