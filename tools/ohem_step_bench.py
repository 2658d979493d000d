#!/usr/bin/env python
"""OHEM cost on the benchmark step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs): prints one JSON line with
  * images/s of NetModel.optimize_parameters() with the plain DSN cross entropy and with `ohem=True` (CriterionOhemDSN);
  * CUDA-event time of the two OHEM threshold passes per step (1/8 grid sample, radix select), measured eagerly on the
    step's logit shape;
  * as context, the reference's host round trip on the same tensors: .cpu() of the full-resolution probabilities, the two
    scipy zooms, np.partition and a .cuda() of the new target.

    python tools/ohem_step_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, BATCH = 512, 1024, 8


def synthetic(seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    images = torch.randn(BATCH, 3, H, W, generator=g)
    labels = torch.randint(0, 19, (BATCH, H, W), generator=g)
    labels[torch.rand(BATCH, H, W, generator=g) < 0.05] = 255
    return images, labels


def step_rate(ohem, steps, warmup):
    import torch
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    margs = make_args(batch_size=BATCH, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", cuda_graph=True, ohem=ohem)
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
    out = {"images_per_s": BATCH * 1e3 / ms, "ms_per_step": ms, "mc_loss": float(model.mc_G_loss)}
    if ohem:
        out.update(threshold=float(model.criterion.last_threshold), kept=float(model.criterion.last_kept))
    del model
    torch.cuda.empty_cache()
    return out


def threshold_passes(reps=50):
    import torch
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    l0 = (torch.randn(BATCH, 65, 129, 20, device="cuda", generator=g) * 2).permute(0, 3, 1, 2)[:, :19]   # the step's pitched logits
    _, labels = synthetic(100)
    labels = labels.cuda()
    mk = 100000 // 64
    for _ in range(3):
        pred, _, nv = ops.ohem_grid_sample(l0, labels, 8, 255)
        ops.ohem_threshold(pred, nv, mk, 0.7)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    grid_ms = sel_ms = 0.0
    for _ in range(reps):
        ev[0].record()
        pred, _, nv = ops.ohem_grid_sample(l0, labels, 8, 255)
        ev[1].record()
        ops.ohem_threshold(pred, nv, mk, 0.7)
        ev[2].record()
        torch.cuda.synchronize()
        grid_ms += ev[0].elapsed_time(ev[1]); sel_ms += ev[1].elapsed_time(ev[2])
    return l0, labels, {"grid_sample_ms": grid_ms / reps, "radix_select_ms": sel_ms / reps, "grid_points": pred.numel()}


def host_round_trip(l0, labels, reps=2):
    """The reference's generate_new_target (utils/criterion.py:50-76) on the same tensors, after an on-GPU softmax(up(l0))."""
    import numpy as np
    import torch
    import torch.nn.functional as F
    from tools import ohem_oracle as O
    dts = []
    for _ in range(reps):
        prob = torch.softmax(F.interpolate(l0.contiguous(), size=(H, W), mode="bilinear", align_corners=True), 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        np_prob, np_target = prob.cpu().numpy(), labels.cpu().numpy()
        t1 = time.perf_counter()
        pred, _ = O.ohem_grid(np_prob, np_target, 8)
        thr = np.float32(O.ohem_threshold(pred, 100000 // 64, 0.7))
        valid = np_target != 255
        p_lab = np.take_along_axis(np_prob, np.where(valid, np_target, 0)[:, None], 1)[:, 0]
        new_target = torch.from_numpy(np.where(valid & (p_lab <= thr), np_target, 255)).cuda()
        torch.cuda.synchronize()
        dts.append((time.perf_counter() - t0, t1 - t0))
        del prob, new_target
    return {"ms": 1e3 * min(d[0] for d in dts), "d2h_ms": 1e3 * min(d[1] for d in dts), "d2h_bytes": BATCH * 19 * H * W * 4,
            "host_threads": os.cpu_count()}


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
    ap.add_argument("--rounds", type=int, default=2, help="plain / ohem measurements, alternated")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    plain, ohem = [], []
    for _ in range(args.rounds):
        plain.append(step_rate(False, args.steps, args.warmup))
        ohem.append(step_rate(True, args.steps, args.warmup))
    l0, labels, passes = threshold_passes()
    host = host_round_trip(l0, labels)
    best_p = min(plain, key=lambda r: r["ms_per_step"]); best_o = min(ohem, key=lambda r: r["ms_per_step"])
    passes["share_of_ohem_step"] = (passes["grid_sample_ms"] + passes["radix_select_ms"]) / best_o["ms_per_step"]
    print(json.dumps({"workload": "batch %d at %dx%d, Pi+Pa+Ho (wgan-gp), CUDA graphs, synthetic inputs" % (BATCH, H, W),
                      "gpu": gpu_info(), "steps": args.steps, "plain": plain, "ohem": ohem,
                      "ohem_over_plain_ms": best_o["ms_per_step"] - best_p["ms_per_step"], "threshold_passes": passes,
                      "reference_host_round_trip": host}))


if __name__ == "__main__":
    main()
