#!/usr/bin/env python
"""Cost of attention transfer and MIMIC on the benchmark step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs): prints one JSON line
with
  * ms per NetModel.optimize_parameters() without the terms and with each of: AT on the PSP features, AT at five levels, MIMIC on the
    PSP features (128 -> 512 adapter), MIMIC on x4 (512 -> 2048 adapter), alternated round by round, and the ms each adds;
  * CUDA-event time of the AT and MSE kernels alone (forward + backward) on the step's own features, to show what the loss passes
    cost beside the adapter's convolutions;
  * the card's name and power limit.

    python tools/feature_kd_step_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.pa_levels_step_bench import BATCH, H, W, gpu_info, synthetic  # noqa: E402

MODES = {"base": {}, "at_psp": dict(at=True), "at_levels5": dict(at=True, lambda_at=[500.0] * 5), "mimic_psp": dict(mimic=True),
         "mimic_x4": dict(mimic=True, lambda_mimic=[0.0, 0.0, 0.0, 1.0])}


def step_ms(mode, steps, warmup):
    import torch
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    torch.cuda.reset_peak_memory_stats()
    margs = make_args(batch_size=BATCH, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", cuda_graph=True, **MODES[mode])
    model = NetModel(margs)
    images, labels = synthetic(100)
    images, labels = images.cuda(), labels.cuda()
    for _ in range(max(warmup, 5)):                                     # 3 eager steps, capture, replays
        model.set_input((images, labels, None, None))
        model.optimize_parameters()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        model.adjust_learning_rate(margs.lr_g, model.G_solver, i)
        model.adjust_learning_rate(margs.lr_d, model.D_solver, i)
        model.set_input((images, labels, None, None))
        model.optimize_parameters()
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / steps
    out = {"ms_per_step": ms, "images_per_s": BATCH * 1e3 / ms, "peak_mem_GB": torch.cuda.max_memory_allocated() / 2 ** 30}
    for term in ("at", "mimic"):
        v = getattr(model, term + "_G_loss")
        if v is not None:
            out[term] = [float(t) for t in v] if isinstance(v, list) else float(v)
    del model
    torch.cuda.empty_cache()
    return out


def kernel_times(reps=20):
    """Eager AT forward + student backward per level, and the MSE forward + backward at the PSP / x4 adapter outputs' shapes."""
    import torch
    from structure_knowledge_distillation_b200 import functions as Fn
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    model = NetModel(make_args(batch_size=BATCH, pi=True, pa=True, ho=False))
    images, labels = synthetic(100)
    model.set_input((images, labels, None, None))
    with torch.no_grad():
        model.forward()
    preds_S, preds_T = model.preds_S, model.preds_T

    def timed(fwd):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        tf = tb = 0.0
        for r in range(reps + 3):
            ev[0].record()
            loss, x = fwd()
            ev[1].record()
            torch.autograd.grad(loss, x)
            ev[2].record()
            torch.cuda.synchronize()
            if r >= 3:
                tf += ev[0].elapsed_time(ev[1]); tb += ev[1].elapsed_time(ev[2])
        return {"fwd_ms": tf / reps, "bwd_ms": tb / reps}

    res = []
    for ind in range(5):
        i = -(ind + 1)
        f = preds_S[i].detach().requires_grad_(True)
        rec = {"term": "at", "level": ind, "channels_S_T": [f.shape[1], preds_T[i].shape[1]], "map": list(f.shape[2:])}
        rec.update(timed(lambda: (Fn.AttentionTransferLoss.apply(f, preds_T[i]), f)))
        res.append(rec)
    for ind in (4, 3):
        i = -(ind + 1)
        t = preds_T[i]
        r = torch.randn_like(t, memory_format=torch.channels_last).requires_grad_(True)
        rec = {"term": "mse", "level": ind, "channels": t.shape[1], "map": list(t.shape[2:])}
        rec.update(timed(lambda: (Fn.MseLoss.apply(r, t), r)))
        res.append(rec)
    del model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2, help="measurements of every mode, alternated")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    runs = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for m in MODES:
            runs[m].append(step_ms(m, args.steps, args.warmup))
    best = {m: min(r["ms_per_step"] for r in rs) for m, rs in runs.items()}
    print(json.dumps({"workload": "batch %d at %dx%d, Pi+Pa+Ho (wgan-gp), CUDA graphs, synthetic inputs" % (BATCH, H, W),
                      "gpu": gpu_info(), "steps": args.steps, "runs": runs,
                      "added_ms": {m: best[m] - best["base"] for m in MODES if m != "base"}, "kernels": kernel_times()}))


if __name__ == "__main__":
    main()
