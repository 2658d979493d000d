#!/usr/bin/env python
"""Cost of the local pair-wise term on the benchmark step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs): prints one JSON line
with
  * ms per NetModel.optimize_parameters() for the default (Pa fully connected on the PSP features at pool_scale 0.5: 9 nodes), local Pa
    on the PSP features at one node per pixel (pool_scale 1/65: 65x129 nodes) with k = 3, 9, 15 and k = 9 at dilation 2, the fully
    connected term at that same scale (the wgmma path, 8 385 nodes), and local Pa on x1 alone at one node per pixel (1/129: 129x257
    nodes, k = 9; no fully connected counterpart: its E would be 35 GB), alternated round by round, and the ms each adds to the default;
  * CUDA-event time of skd_pairwise_local_fwd and skd_pairwise_local_bwd alone on the step's own pooled features, with the FLOP rate of
    the connected pairs' dot products (2 * N * P * (C_S + C_T) forward, 2 * N * P * C_S backward);
  * the card's name and power limit.

    python tools/pa_local_step_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.pa_levels_step_bench import BATCH, H, W, gpu_info, synthetic  # noqa: E402

PSP_1PX, X1_1PX = 1.0 / 65, 1.0 / 129
MODES = {"default": {},
         "local_psp_k3": dict(pool_scale=PSP_1PX, pa_window=3), "local_psp_k9": dict(pool_scale=PSP_1PX, pa_window=9),
         "local_psp_k15": dict(pool_scale=PSP_1PX, pa_window=15),
         "local_psp_k9_d2": dict(pool_scale=PSP_1PX, pa_window=9, pa_dilation=2),
         "global_psp_1px": dict(pool_scale=PSP_1PX),
         "local_x1_k9": dict(lambda_pa=[0.5], pool_scale=[X1_1PX], pa_window=[9])}


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
    pa = model.pa_G_loss
    out = {"ms_per_step": ms, "images_per_s": BATCH * 1e3 / ms, "peak_mem_GB": torch.cuda.max_memory_allocated() / 2 ** 30,
           "pa": [float(t) for t in pa] if isinstance(pa, list) else float(pa)}
    del model
    torch.cuda.empty_cache()
    return out


def kernel_times(reps=20):
    """The two kernels alone, on the pooled rows of one eager forward's PSP features (65x129 nodes) and x1 (129x257 nodes)."""
    import torch
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    model = NetModel(make_args(batch_size=BATCH, pi=True, pa=True, ho=False))
    images, labels = synthetic(100)
    model.set_input((images, labels, None, None))
    with torch.no_grad():
        model.forward()
    L = lib()
    res = []
    for level, ind, ks in (("psp", -5, ((3, 1), (9, 1), (15, 1), (9, 2))), ("x1", -1, ((9, 1),))):
        fS, fT = model.preds_S[ind].detach(), model.preds_T[ind]
        pS, _, rS = ops.pairwise_pool(fS, 1, 1, False)
        pT, _, rT = ops.pairwise_pool(fT, 1, 1, False)
        n, cs, h, w = fS.shape
        ct = fT.shape[1]
        g = torch.ones((), device="cuda")
        for k, d in ks:
            E = torch.empty((n, h * w, k * k), device="cuda")
            parts = torch.empty(L.skd_pairwise_local_partials(n, h, w, k, d), device="cuda", dtype=torch.float64)
            loss = torch.empty((), device="cuda")
            dp = torch.empty_like(pS)
            st = torch.cuda.current_stream().cuda_stream
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            tf = tb = 0.0
            for r in range(reps + 3):
                ev[0].record()
                L.skd_pairwise_local_fwd(n, h, w, cs, ct, pS.data_ptr(), pT.data_ptr(), rS.data_ptr(), rT.data_ptr(), k, d, E.data_ptr(),
                                         loss.data_ptr(), parts.data_ptr(), st)
                ev[1].record()
                L.skd_pairwise_local_bwd(n, h, w, cs, E.data_ptr(), pS.data_ptr(), rS.data_ptr(), k, d, g.data_ptr(), dp.data_ptr(), st)
                ev[2].record()
                torch.cuda.synchronize()
                if r >= 3:
                    tf += ev[0].elapsed_time(ev[1]); tb += ev[1].elapsed_time(ev[2])
            tf, tb = tf / reps, tb / reps
            pairs = ops.pairwise_local_pairs(h, w, k, d)
            res.append({"level": level, "grid": [h, w], "channels_S_T": [cs, ct], "window": k, "dilation": d, "fwd_ms": tf, "bwd_ms": tb,
                        "fwd_TFLOPs": 2.0 * n * pairs * (cs + ct) / tf / 1e9, "bwd_TFLOPs": 2.0 * n * pairs * cs / tb / 1e9,
                        "E_MB": E.numel() * 4 / 2 ** 20})
            del E
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
                      "added_ms": {m: best[m] - best["default"] for m in MODES if m != "default"}, "kernels": kernel_times()}))


if __name__ == "__main__":
    main()
