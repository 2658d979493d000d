#!/usr/bin/env python
"""Cost of multi-level pair-wise distillation on the benchmark step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs): prints
one JSON line with
  * images/s of NetModel.optimize_parameters() with the scalar Pa term (preds[-5], pool_scale 0.5) and with five levels
    (lambda_pa [0.5]*5, pool_scale [0.5]*5), alternated in this one call, and the peak device memory of each;
  * CUDA-event time of each level's Pa forward and feature backward at scale 0.5, measured eagerly on the step's own features;
  * the same for the PSP level at scale 1/65 (65x129 = 8 385 nodes, the wgmma regime), with the size of its stored E;
  * the card's name and power limit.

    python tools/pa_levels_step_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, BATCH = 512, 1024, 8
MODES = {"scalar": dict(lambda_pa=0.5, pool_scale=0.5), "levels5": dict(lambda_pa=[0.5] * 5, pool_scale=[0.5] * 5)}


def synthetic(seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    images = torch.randn(BATCH, 3, H, W, generator=g)
    labels = torch.randint(0, 19, (BATCH, H, W), generator=g)
    labels[torch.rand(BATCH, H, W, generator=g) < 0.05] = 255
    return images, labels


def step_rate(mode, steps, warmup):
    import torch
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    torch.cuda.reset_peak_memory_stats()
    margs = make_args(batch_size=BATCH, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", cuda_graph=True, **MODES[mode])
    model = NetModel(margs)
    images, labels = synthetic(100)
    images, labels = images.cuda(), labels.cuda()
    for i in range(max(warmup, 5)):                                     # 3 eager steps, capture, replays
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
    pa = model.pa_G_loss
    out = {"images_per_s": BATCH * 1e3 / ms, "ms_per_step": ms, "peak_mem_GB": torch.cuda.max_memory_allocated() / 2 ** 30,
           "pa": [float(v) for v in pa] if isinstance(pa, list) else float(pa)}
    del model
    torch.cuda.empty_cache()
    return out


def level_times(reps=20):
    """Eager forward + feature backward of one Pa criterion per level on the features of one benchmark-shaped forward."""
    import torch
    from structure_knowledge_distillation_b200 import functions as Fn
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.criterion import CriterionPairWiseforWholeFeatAfterPool
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    model = NetModel(make_args(batch_size=BATCH, pi=True, pa=True, ho=False))
    images, labels = synthetic(100)
    model.set_input((images, labels, None, None))
    with torch.no_grad():
        model.forward()
    preds_S, preds_T = list(model.preds_S), model.preds_T
    res = []
    for ind, scale in [(0, 0.5), (1, 0.5), (2, 0.5), (3, 0.5), (4, 0.5), (4, 1.0 / 65)]:
        i = -(ind + 1)
        crit = CriterionPairWiseforWholeFeatAfterPool(scale=scale, feat_ind=i)
        f = preds_S[i].detach().requires_grad_(True)
        S = list(preds_S); S[i] = f
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        fwd = bwd = 0.0
        for r in range(reps + 3):
            ev[0].record()
            loss = crit(S, preds_T)
            ev[1].record()
            torch.autograd.grad(loss, f)
            ev[2].record()
            torch.cuda.synchronize()
            if r >= 3:                                                  # first launches warm modules and allocations
                fwd += ev[0].elapsed_time(ev[1]); bwd += ev[1].elapsed_time(ev[2])
        h, w = preds_T[i].shape[2:]
        ph, pw = int(h * scale), int(w * scale)
        nodes = -(-h // ph) * -(-w // pw)
        wgmma = nodes >= Fn.PairWiseLoss.TCGEN05_MIN_NODES
        res.append({"level": ind, "feature": ("x1", "x2", "x3", "x4", "psp")[ind], "scale": scale, "map": [h, w],
                    "channels_S_T": [f.shape[1], preds_T[i].shape[1]], "nodes": nodes, "path": "wgmma" if wgmma else "simt",
                    "E_GB": BATCH * nodes * nodes * 4 / 2 ** 30 if wgmma else None,
                    "fwd_ms": fwd / reps, "bwd_ms": bwd / reps, "ms": (fwd + bwd) / reps})
        del loss
    del model
    torch.cuda.empty_cache()
    return res


def gpu_info():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as ex:                                              # noqa: BLE001
        return {"error": repr(ex)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2, help="scalar / five-level measurements, alternated")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    runs = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for m in MODES:
            runs[m].append(step_rate(m, args.steps, args.warmup))
    best = {m: min(r, key=lambda x: x["ms_per_step"]) for m, r in runs.items()}
    print(json.dumps({"workload": "batch %d at %dx%d, Pi+Pa+Ho (wgan-gp), CUDA graphs, synthetic inputs" % (BATCH, H, W),
                      "gpu": gpu_info(), "steps": args.steps, "runs": runs,
                      "levels5_over_scalar_ms": best["levels5"]["ms_per_step"] - best["scalar"]["ms_per_step"],
                      "per_level": level_times()}))


if __name__ == "__main__":
    main()
