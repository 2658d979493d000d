#!/usr/bin/env python
"""Cost of channel-wise distillation (CWD) on the benchmark step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs): prints one JSON
line with
  * ms per NetModel.optimize_parameters() and peak allocation without CWD and with each of: CWD on the logits, logits + the PSP level
    (128 -> 512 adapter), logits + x4 (512 -> 2048 adapter), x1 alone (256 -> 256 adapter), alternated round by round, and the ms each
    adds;
  * CUDA-event times of the CWD forward and backward alone, launched through the C ABI on preallocated buffers, at the logits
    (19 of 20 channels, 65x129), the PSP adapter output (512 channels, 65x129) and x1 (256 channels, 129x257), with the bytes the
    algorithm must move (forward: each map read twice; backward: S and T read, dS written) and the achieved GB/s beside the
    3.35 TB/s data-sheet rate;
  * the card's name and power limit.

    python tools/cwd_step_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.pa_levels_step_bench import BATCH, H, W, gpu_info, synthetic  # noqa: E402

MODES = {"none": {}, "cwd_logits": dict(cwd=True), "cwd_logits_psp": dict(cwd=True, lambda_cwd_feat=1.0),
         "cwd_logits_x4": dict(cwd=True, lambda_cwd_feat=[0.0, 0.0, 0.0, 1.0]),
         "cwd_x1": dict(cwd=True, lambda_cwd=0.0, lambda_cwd_feat=[1.0])}
HBM_GBPS = 3350.0
# (name, channels, row pitch, H, W) of the maps the step's CWD terms read at batch 8
KERNEL_SHAPES = [("logits", 19, 20, 65, 129), ("psp_adapter", 512, 512, 65, 129), ("x1", 256, 256, 129, 257)]


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
    v = model.cwd_G_loss
    if v is not None:
        out["cwd"] = [float(t) for t in v] if isinstance(v, list) else float(v)
    del model
    torch.cuda.empty_cache()
    return out


def kernel_times(reps=50):
    """skd_cwd_fwd / skd_cwd_bwd alone on random NHWC maps of the step's shapes (teacher and student at the same pitch)."""
    import torch
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    res = []
    for name, c, pitch, h, w in KERNEL_SHAPES:
        g = torch.Generator(device="cuda").manual_seed(1)
        S = (torch.randn(BATCH, h, w, pitch, generator=g, device="cuda") * 3).permute(0, 3, 1, 2)[:, :c]
        T = (torch.randn(BATCH, h, w, pitch, generator=g, device="cuda") * 3).permute(0, 3, 1, 2)[:, :c]
        dS = torch.empty_strided(S.shape, S.stride(), device="cuda")
        loss = torch.empty((), device="cuda")
        lse = torch.empty((2, BATCH, c), device="cuda", dtype=torch.float64)
        ws = torch.empty(L.skd_cwd_workspace(BATCH, c, h * w), device="cuda", dtype=torch.float64)
        gout = torch.ones((), device="cuda")
        sS, sT, sD = ops.pixel_strides(S), ops.pixel_strides(T), ops.pixel_strides(dS)

        def fwd():
            L.skd_cwd_fwd(BATCH, c, h * w, S.data_ptr(), *sS, T.data_ptr(), *sT, 4.0, loss.data_ptr(), lse.data_ptr(), ws.data_ptr(), st)

        def bwd():
            L.skd_cwd_bwd(BATCH, c, h * w, S.data_ptr(), *sS, T.data_ptr(), *sT, 4.0, lse.data_ptr(), gout.data_ptr(), dS.data_ptr(),
                          *sD, st)

        def timed(fn):
            for _ in range(5):
                fn()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            for _ in range(reps):
                fn()
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]) / reps

        fms, bms = timed(fwd), timed(bwd)
        map_bytes = BATCH * c * h * w * 4
        fb, bb = 4 * map_bytes, 3 * map_bytes                  # forward: S and T read twice; backward: S, T read, dS written
        res.append({"map": name, "shape": [BATCH, c, h, w], "pitch": pitch, "fwd_ms": fms, "bwd_ms": bms, "fwd_bytes": fb, "bwd_bytes": bb,
                     "fwd_GBps": fb / fms / 1e6, "bwd_GBps": bb / bms / 1e6, "fwd_share_of_3350GBps": fb / fms / 1e6 / HBM_GBPS,
                     "bwd_share_of_3350GBps": bb / bms / 1e6 / HBM_GBPS})
        del S, T, dS, ws
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
                      "added_ms": {m: best[m] - best["none"] for m in MODES if m != "none"}, "kernels": kernel_times()}))


if __name__ == "__main__":
    main()
