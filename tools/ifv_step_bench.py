#!/usr/bin/env python
"""Cost of intra-class feature variation distillation (IFV) on the benchmark step (batch 8 at 512x1024, Pi+Pa+Ho wgan-gp, CUDA graphs):
prints one JSON line with
  * ms per NetModel.optimize_parameters() and peak allocation without IFV and with each of: the PSP level (128 student against 512
    teacher channels), all five levels, x1 alone (64 against 256), alternated round by round, and the ms each adds;
  * CUDA-event times of the IFV forward and backward alone, launched through the C ABI on preallocated buffers, at the PSP level
    (65x129) and at x1 (129x257), 19 classes, with the bytes the algorithm must move (forward: each map read twice; backward: S read
    twice, dS written) and the achieved GB/s beside the 3.35 TB/s data-sheet rate;
  * the card's name and power limit.

    python tools/ifv_step_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.pa_levels_step_bench import BATCH, H, W, gpu_info, synthetic  # noqa: E402

MODES = {"none": {}, "ifv_psp": dict(ifv=True), "ifv_levels": dict(ifv=True, lambda_ifv=[200.0] * 5),
         "ifv_x1": dict(ifv=True, lambda_ifv=[200.0])}
HBM_GBPS = 3350.0
K = 19
# (name, student channels, teacher channels, h, w) of the maps the step's IFV terms read at batch 8
KERNEL_SHAPES = [("psp", 128, 512, 65, 129), ("x1", 64, 256, 129, 257)]


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
    v = model.ifv_G_loss
    if v is not None:
        out["ifv"] = [float(t) for t in v] if isinstance(v, list) else float(v)
    del model
    torch.cuda.empty_cache()
    return out


def kernel_times(reps=50):
    """skd_ifv_fwd / skd_ifv_bwd alone on random dense NHWC maps of the step's shapes with 19-class labels (5 % ignored)."""
    import torch
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    L, st = lib(), torch.cuda.current_stream().cuda_stream
    res = []
    for name, cs, ct, h, w in KERNEL_SHAPES:
        g = torch.Generator(device="cuda").manual_seed(1)
        S = torch.randn(BATCH, h, w, cs, generator=g, device="cuda").permute(0, 3, 1, 2)
        T = torch.randn(BATCH, h, w, ct, generator=g, device="cuda").permute(0, 3, 1, 2)
        labels = torch.randint(0, K, (BATCH, H, W), generator=g, device="cuda")
        labels[torch.rand(BATCH, H, W, generator=g, device="cuda") < 0.05] = 255
        lab = ops.labels_nearest(labels, h, w)
        dS = torch.empty_like(S)
        loss = torch.empty((), device="cuda")
        PS = torch.empty((BATCH, K, cs), device="cuda")
        stats = torch.empty((3, BATCH, K), device="cuda", dtype=torch.float64)
        pix = torch.empty((3, BATCH, h * w), device="cuda")
        ws = torch.empty(L.skd_ifv_workspace(BATCH, h * w, K, cs, ct), device="cuda", dtype=torch.float64)
        gout = torch.ones((), device="cuda")
        (sn, sp), (tn, tp) = ops._row_strides(S), ops._row_strides(T)

        def fwd():
            L.skd_ifv_fwd(BATCH, h * w, K, lab.data_ptr(), S.data_ptr(), cs, sn, sp, T.data_ptr(), ct, tn, tp, loss.data_ptr(), PS.data_ptr(),
                          stats.data_ptr(), pix.data_ptr(), ws.data_ptr(), st)

        def bwd():
            L.skd_ifv_bwd(BATCH, h * w, K, lab.data_ptr(), S.data_ptr(), cs, sn, sp, PS.data_ptr(), stats.data_ptr(), pix.data_ptr(),
                          gout.data_ptr(), dS.data_ptr(), sn, sp, ws.data_ptr(), st)

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

        fms = timed(fwd)
        bms = timed(bwd)
        s_bytes, t_bytes = BATCH * cs * h * w * 4, BATCH * ct * h * w * 4
        fb, bb = 2 * (s_bytes + t_bytes), 3 * s_bytes           # forward: S and T read twice; backward: S read twice, dS written
        res.append({"map": name, "S": [BATCH, cs, h, w], "T": [BATCH, ct, h, w], "classes": K, "fwd_ms": fms, "bwd_ms": bms,
                    "fwd_bytes": fb, "bwd_bytes": bb, "fwd_GBps": fb / fms / 1e6, "bwd_GBps": bb / bms / 1e6,
                    "fwd_share_of_3350GBps": fb / fms / 1e6 / HBM_GBPS, "bwd_share_of_3350GBps": bb / bms / 1e6 / HBM_GBPS})
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
