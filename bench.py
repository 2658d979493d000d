#!/usr/bin/env python
"""bench.py -- distillation-step images/sec at 512x1024 (Pi+Pa+Ho), BASELINE.json's metric.

  python bench.py --gpus N --steps K --warmup W            our arm  (one process per GPU; under torchrun for N > 1)
  python bench.py --impl reference ...                      the reference's own algorithm on the box's host cores

One "step" = NetModel.optimize_parameters(): frozen PSPNet-101 teacher forward, ResNet18-PSP student forward, CE+Pi+Pa+Ho
losses, student backward, SGD step, discriminator step (WGAN-GP) -- nothing skipped.  Workload = BASELINE.json
configs[2]: batch 8 per GPU at 512x1024, synthetic tensors, random-init weights (no dataset / checkpoints offline).

Printed JSON (rank 0, one line):
  value  images/s with the batch already resident in HBM (CUDA events, max over ranks);
  e2e    same step through the public API from pinned HOST buffers: per step an H2D copy of images+labels and a D2H read
         of the loss inside the timed region;
  roofline  the dominant kernel (wgmma implicit-GEMM conv, fwd+dgrad launches): algorithmic FLOP / CUDA-event time of
            every launch of it inside the timed region, against the tensor peak;
  cpu_baseline  oracle/port.py (CPU restatement pinned to the reference) on a bounded sample, N=1 rank 0 only.

--dump-outputs DIR writes, after the timed steps, what the last timed step computed (rank 0) as DIR/<name>.npy: the step's losses
(float64), the student's and the teacher's main logits, and a fixed seeded sample of the updated student and discriminator
parameters (float32).  Inputs and initial weights are seeded, so two builds run with the same arguments can be compared output for
output.  Every reduction on the timed path adds in a fixed order, so a build reproduces its own dump bit for bit; between two builds
that sum in different orders, the random-init training amplifies last-bit differences from step to step, so compare those with
few steps (--steps 1).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H, W, BATCH_PER_GPU = 512, 1024, 8
METRIC = "distillation-step images/sec at 512x1024 (Pi+Pa+Ho)"
WORKLOAD = "BASELINE.json configs[2]: ResNet18-PSP student + PSPNet-101 teacher, Pi+Pa+Ho (wgan-gp), batch 8/GPU at 512x1024, pool_scale 0.5"
# algorithmic conv GFLOP per image: teacher forward, student forward (SURVEY.md 8d: hooks on the reference model)
FLOP_T, FLOP_S, FLOP_STEM1 = 1149.9e9, 251.7e9, 0.45e9


def select_config(cfg):
    """--config 4: BASELINE.json configs[3] shape -- 360x480 (CamVid crops, 46x61 logits), batch 16 per GPU, Pi+Pa+Ho.  The student is
    the ResNet18-PSP one (the reference ships no ESPNet source: SURVEY.md 8c); the discriminator runs with its size-aware head."""
    global H, W, BATCH_PER_GPU, METRIC, WORKLOAD, FLOP_T, FLOP_S, FLOP_STEM1
    if cfg == 4:
        H, W, BATCH_PER_GPU = 360, 480, 16
        METRIC = "distillation-step images/sec at 360x480 (Pi+Pa+Ho)"
        WORKLOAD = ("BASELINE.json configs[3] shape: ResNet18-PSP student (no ESPNet source in the reference) + PSPNet-101 teacher, Pi+Pa+Ho (wgan-gp), "
                    "batch 16/GPU at 360x480, pool_scale 0.5, size-aware discriminator head")
        FLOP_T, FLOP_S, FLOP_STEM1 = 384.7e9, 84.0e9, 0.45e9 * (360 * 480) / (512 * 1024)


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d["hbm_gbs"], bf16=d["bf16_tflops"], bf16_sus=d.get("bf16_tflops_sustained", d["bf16_tflops"]), src="measured")
    return dict(hbm=3350.0, bf16=989.0, bf16_sus=989.0, src="H100 SXM data sheet")


class ClockSampler:
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True); self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if not self.proc:
            return dict(sm_mhz=None, sm_max_mhz=None, reasons=["nvidia-smi unavailable"])
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for r in self.rows if len(r) >= 7 for i in range(4) if r[3 + i].lower().startswith("active")})
        return dict(sm_mhz=statistics.median(sm) if sm else None, sm_max_mhz=max(mx) if mx else None, reasons=reasons,
                    samples=len(sm))


def synthetic(batch, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    images = torch.randn(batch, 3, H, W, generator=g)
    labels = torch.randint(0, 19, (batch, H, W), generator=g)
    labels[torch.rand(batch, H, W, generator=g) < 0.05] = 255
    return images, labels


# ------------------------------------------------------------------------------------------------------------------
def run_reference(args, rank, world):
    """The reference's own algorithm (oracle/port.py: CPU restatement pinned against the unmodified reference by golden fixtures,
    so the reference tree itself is not needed here) on all host threads.  Bounded sample: batch 1 per step."""
    if rank != 0:
        return
    import torch
    from oracle import cases, port
    if args.ref_device == "cuda":
        return run_reference_cuda(args)
    cores = _cpu_threads()
    torch.set_num_threads(cores)
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    g_opt, d_opt = port.make_optimizers(student, D, cfg)
    images, labels = synthetic(1, 0)
    alpha = torch.rand(1, 1, 1, 1)
    steps, warm = max(1, min(args.steps, 3)), max(1, min(args.warmup, 1))
    for _ in range(warm):
        port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
    dts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
        dts.append(time.perf_counter() - t0)
    dt = sum(dts) / steps
    v = 1.0 / dt
    sample = "batch 1 of the same 512x1024 Pi+Pa+Ho(wgan-gp) step, %d timed steps (%s s) after %d warm-up, fp32 torch CPU, %d threads (cap; %s logical CPUs)" % (
        steps, "/".join("%.2f" % d for d in dts), warm, cores, os.cpu_count())
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": v, "unit": "images/s", "n_gpus": args.gpus, "steps": steps, "warmup": warm,
        "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "BASELINE.json configs[2]: ResNet18 student + PSPNet-101 teacher, Pi+Pa+Ho, 512x1024 (bounded sample: batch 1)"},
        "cpu_baseline": {"value": v, "unit": "images/s", "cores": cores, "kind": "port", "sample": sample},
        "e2e": {"value": v, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))


def run_reference_cuda(args):
    """Not the contract's reference arm (that is the CPU leg above): the same restatement with its torch ops placed on cuda:0
    -- cuDNN/cuBLAS eager, NCHW fp32, full batch 8 -- i.e. what the reference's stock code path costs on this box.  Printed as
    context for the headline; `--ref-tf32 0` disables TF32 in cuDNN (torch's default allows it)."""
    import torch
    from oracle import cases, port
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = True                                    # train_and_eval.py sets cudnn.benchmark
    torch.backends.cudnn.allow_tf32 = bool(args.ref_tf32)
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    teacher.to(dev); student.to(dev); D.to(dev)
    g_opt, d_opt = port.make_optimizers(student, D, cfg)
    images, labels = synthetic(BATCH_PER_GPU, 0)
    images, labels = images.to(dev), labels.to(dev)
    alpha = torch.rand(BATCH_PER_GPU, 1, 1, 1, device=dev)
    steps, warm = args.steps, max(3, args.warmup)
    for _ in range(warm):
        port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
    e.record(); torch.cuda.synchronize()
    ms = s.elapsed_time(e) / steps
    print(json.dumps({
        "impl": "reference", "device": "cuda (torch eager: cuDNN/cuBLAS, tf32 %s)" % ("allowed" if args.ref_tf32 else "off"),
        "metric": METRIC, "value": BATCH_PER_GPU * 1e3 / ms, "unit": "images/s", "n_gpus": 1, "steps": steps, "warmup": warm,
        "ms_per_step": ms, "higher_is_better": True, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "BASELINE.json configs[2]: ResNet18 student + PSPNet-101 teacher, Pi+Pa+Ho, 512x1024, batch %d, inputs resident" % BATCH_PER_GPU},
        "peak_mem_gb": torch.cuda.max_memory_allocated() / 2**30}))


def _cpu_threads():
    # torch's CPU convolutions stop scaling (and on 100+ thread boxes get much slower) for a batch-1 step: cap at 32 threads
    return min(os.cpu_count() or 1, 32)


def cpu_baseline_leg(timed=3):
    """oracle/port.py on the host cores: median of `timed` steps after one warm-up (single steps scatter by +-50 %)."""
    import torch
    from oracle import cases, port
    cores = _cpu_threads()
    torch.set_num_threads(cores)
    cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
    teacher, student, D = cases.build_models(seed=0, with_D=True)
    g_opt, d_opt = port.make_optimizers(student, D, cfg)
    images, labels = synthetic(1, 0)
    alpha = torch.rand(1, 1, 1, 1)
    port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
    dts = []
    for _ in range(timed):
        t0 = time.perf_counter()
        port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
        dts.append(time.perf_counter() - t0)
    dt = statistics.median(dts)
    return {"value": 1.0 / dt, "unit": "images/s", "cores": cores, "host_logical_cpus": os.cpu_count(), "kind": "port",
            "step_seconds": [round(d, 3) for d in dts],
            "sample": "oracle/port.py (CPU restatement of the reference step), batch 1 @512x1024 Pi+Pa+Ho, median of %d timed steps after 1 warm-up, "
                      "%d torch threads (cap; the box has %s logical CPUs)" % (timed, cores, os.cpu_count())}


def torch_cuda_eager_context(batch=4, steps=5):
    """Context only (not the contract's reference arm): the same restatement with its torch ops on cuda:0 -- cuDNN / cuBLAS eager, TF32
    allowed (torch's default), i.e. what the reference's stock code path costs on this GPU.  Batch 4 bounds its memory."""
    import torch
    from oracle import cases, port
    try:
        dev = torch.device("cuda", 0)
        torch.backends.cudnn.benchmark = True
        cfg = port.StepConfig(pi=True, pa=True, ho=True, adv_type="wgan-gp")
        teacher, student, D = cases.build_models(seed=0, with_D=True)
        teacher.to(dev); student.to(dev); D.to(dev)
        g_opt, d_opt = port.make_optimizers(student, D, cfg)
        images, labels = synthetic(batch, 0)
        images, labels = images.to(dev), labels.to(dev)
        alpha = torch.rand(batch, 1, 1, 1, device=dev)
        for _ in range(3):
            port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            port.distill_step(teacher, student, D, images, labels, cfg, g_opt, d_opt, gp_alpha=alpha)
        e.record(); torch.cuda.synchronize()
        ms = s.elapsed_time(e) / steps
        out = {"value": batch * 1e3 / ms, "unit": "images/s", "ms_per_step": ms, "batch": batch,
               "what": "oracle/port.py with its torch ops on cuda:0 (cuDNN/cuBLAS eager, TF32 allowed): context, not the reference arm",
               "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}
        del teacher, student, D, g_opt, d_opt
        torch.cuda.empty_cache()
        return out
    except Exception as ex:                                                # noqa: BLE001
        return {"error": repr(ex)[:200]}


DUMP_PARAM_SAMPLE = 1 << 20          # parameters per model kept by --dump-outputs (a fixed, seeded sample; 64 MB cap on the whole dump)


def dump_outputs(model, out_dir):
    """The arrays a caller of NetModel.optimize_parameters() receives from one step: losses, logits, updated parameters."""
    import numpy as np
    import torch
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    names = ["mc_G_loss", "pi_G_loss", "pa_G_loss", "G_loss", "D_loss"]
    arrays = {"losses": np.array([float(getattr(model, n)) for n in names], dtype=np.float64),
              "student_logits": model.preds_S[0].detach().float().cpu().numpy(),
              "teacher_logits": model.preds_T[0].detach().float().cpu().numpy()}
    for key, solver in (("student_params", model.G_solver), ("discriminator_params", model.D_solver)):
        flat = solver.flat_p.detach()
        if flat.numel() > DUMP_PARAM_SAMPLE:
            g = torch.Generator().manual_seed(0)
            idx = torch.randperm(flat.numel(), generator=g)[:DUMP_PARAM_SAMPLE].sort().values
            flat = flat[idx.to(flat.device)]
        arrays[key + "_sample" if flat.numel() < solver.flat_p.numel() else key] = flat.float().cpu().numpy()
    total = sum(a.nbytes for a in arrays.values())
    assert total <= 64 << 20, total
    for k, a in arrays.items():
        np.save(os.path.join(out_dir, k + ".npy"), a)


# ------------------------------------------------------------------------------------------------------------------
def run_ours(args, rank, local_rank, world):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args

    torch.manual_seed(0)                                          # identical replicas on every rank
    margs = make_args(batch_size=BATCH_PER_GPU, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", gpu_num=world,
                      cuda_graph=not args.no_graph, allreduce_buckets=args.allreduce_buckets, allreduce=args.allreduce)
    model = NetModel(margs)
    # eval-mode BN of the frozen teacher must not be the identity (SURVEY.md §8d)
    g = torch.Generator(device="cuda").manual_seed(1)
    for m in model.teacher.modules():
        if hasattr(m, "running_var"):
            m.running_mean.copy_(torch.randn(m.running_mean.shape, device="cuda", generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.running_var.shape, device="cuda", generator=g) + 0.5)
    images, labels = synthetic(BATCH_PER_GPU, 100 + rank)
    pin_i, pin_l = images.pin_memory(), labels.pin_memory()
    dev_i, dev_l = images.cuda(), labels.cuda()
    L = lib()

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(k, body):
        barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for i in range(k):
            body(i)
        e.record()
        barrier()
        ms = torch.tensor([s.elapsed_time(e)], device="cuda")
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms)

    def step_resident(i):
        model.adjust_learning_rate(margs.lr_g, model.G_solver, i)
        model.adjust_learning_rate(margs.lr_d, model.D_solver, i)
        model.set_input((dev_i, dev_l, None, None))                # the batch is already in HBM: set_input() only moves it device -> device
        model.optimize_parameters()

    sink = []

    def step_e2e(i):
        # the loop a training script runs through the public API, software-pipelined by one batch: launch step i, hand the NEXT batch to
        # set_input() (with captured graphs it goes to staging buffers on a copy stream, i.e. under step i's kernels), then read step i's
        # loss.  Every timed step still contains one host -> device copy of a full batch from pinned memory and one device -> host read.
        model.adjust_learning_rate(margs.lr_g, model.G_solver, i)
        model.adjust_learning_rate(margs.lr_d, model.D_solver, i)
        if i == 0:
            model.set_input((pin_i, pin_l, None, None))           # the first batch of the timed region
        model.optimize_parameters()
        model.set_input((pin_i, pin_l, None, None))               # H2D of the next batch from pinned host memory, every step
        sink.append(float(model.G_loss))                          # D2H read of this step's loss

    use_graph = not args.no_graph
    n_warm = max(args.warmup, 5 if use_graph else 3)              # graphs: 3 eager steps, 1 capture step, >=1 replay
    launches_per_step = 0
    for i in range(n_warm):
        l0 = L.skd_kernel_launches()
        step_resident(i)
        if i == 1:
            launches_per_step = L.skd_kernel_launches() - l0      # our kernels per step, counted on an eager step

    clocks = ClockSampler(local_rank)
    if rank == 0:
        clocks.start()
    ms = timed(args.steps, step_resident)
    clk = clocks.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(model, args.dump_outputs)
    ms_e2e = timed(args.steps, step_e2e)
    launches = launches_per_step * args.steps

    # roofline pass: the same steps executed eagerly with a CUDA-event pair around every wgmma conv launch
    # (events recorded inside a captured graph cannot be timed)
    conv_log = []
    model._graphs = None
    model.overlap_streams = False                                  # one stream: an event pair must bracket ONE kernel, not its neighbours on other streams
    ops.CONV_EVENT_LOG = conv_log                                  # ops.conv2d_fwd records (start, end, flops) per wgmma launch
    ms_eager = timed(args.steps, step_resident)
    ops.CONV_EVENT_LOG = None

    total_images = BATCH_PER_GPU * world * args.steps
    value = total_images / (ms / 1e3)
    e2e = total_images / (ms_e2e / 1e3)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    peaks = _peaks()
    tf32_peak = peaks["bf16_sus"] / 2.0                            # wgmma tf32 issues at half the bf16 rate
    wg_log = [r for r in conv_log if r[3][0] == "wgrad"]
    all_log = conv_log
    conv_log = [r for r in conv_log if r[3][0] in ("fwd", "dgrad", "fwd3x")]         # the dominant kernel: conv_fwd_sm90_kernel (fwd + dgrad)
    conv_ms = sum(r[0].elapsed_time(r[1]) for r in conv_log)
    conv_flop = sum(r[2] for r in conv_log)
    wg_ms = sum(r[0].elapsed_time(r[1]) for r in wg_log)
    wg_flop = sum(r[2] for r in wg_log)
    if args.conv_table:
        import collections
        agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
        for r in all_log:
            a = agg[r[3]]; a[0] += 1; a[1] += r[0].elapsed_time(r[1]); a[2] += r[2]
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])[:40]:
            print("CONV %-48s n=%3d  %7.3f ms/step  %6.0f TF" % (k, v[0] // args.steps, v[1] / args.steps, v[2] / max(v[1], 1e-9) / 1e9), file=sys.stderr)
    achieved = conv_flop / (conv_ms * 1e-3) / 1e12 if conv_ms > 0 else 0.0
    # whole step: algorithmic conv FLOP of one image (SURVEY.md §8d, hooks on the reference model) x batch, over the TIMED (graph) step
    step_flop = (FLOP_T + FLOP_S + 2 * FLOP_S - FLOP_STEM1) * BATCH_PER_GPU
    out = {
        "metric": METRIC, "value": value, "unit": "images/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "tf32",
        "data": "synthetic",
        "config": {"workload": WORKLOAD,
                   "global_batch": BATCH_PER_GPU * world, "parallelism": "dp%d" % world, "gradient_exchange": (args.allreduce if world > 1 else "none"),
                   "precision": "fp32 storage; TF32 tensor-core operands (round-to-nearest by TMA), fp32 accumulate; student stem, layer1 and layer2 forward in split-precision 3xTF32",
                   "cuda_graph": bool(use_graph), "launch_count_note": "gpu_launches = our kernels counted on an eager step x steps (graph replays re-issue the same launches)",
                   "l2": "per-step working set (activations ~10 GB) is far larger than the 50 MB L2: no flush needed"},
        "e2e": {"value": e2e, "unit": "images/s", "h2d_bytes_per_step": pin_i.numel() * 4 + pin_l.numel() * 8, "d2h_bytes_per_step": 4,
                "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": int(launches),
        "clocks": clk,
        "roofline": {"bound": "tensor", "kernel": "conv_fwd_sm90_kernel (wgmma implicit GEMM: teacher fwd, student fwd, student dgrad)",
                     "achieved": achieved, "peak": tf32_peak, "unit": "TFLOP/s", "frac": achieved / tf32_peak if tf32_peak else None,
                     "flop_counting": "algorithmic 2*N*OH*OW*Cout*Cin*KH*KW per launch; split-precision (3xTF32) launches are counted ONCE",
                     "peak_source": "%s bf16 peak / 2 (TF32 operands)" % peaks["src"], "traffic": None,
                     "launches_timed": len(conv_log), "share_of_eager_step": conv_ms / ms_eager if ms_eager else None,
                     "wgrad_kernel": {"achieved": wg_flop / (wg_ms * 1e-3) / 1e12 if wg_ms > 0 else None,
                                      "frac": (wg_flop / (wg_ms * 1e-3) / 1e12) / tf32_peak if wg_ms > 0 and tf32_peak else None,
                                      "share_of_eager_step": wg_ms / ms_eager if ms_eager else None},
                     "whole_step_frac": step_flop / ((ms / args.steps) * 1e-3) / 1e12 / tf32_peak if tf32_peak else None,
                     "whole_step_note": "algorithmic conv FLOP of the step (%.2f TFLOP at batch %d, SURVEY.md 8d) / timed ms_per_step / peak: everything that is "
                                        "not a tensor-core convolution (ABN, losses, discriminator, SGD, glue) counts against it" % (step_flop / 1e12, BATCH_PER_GPU),
                     "measured_in": "per-launch CUDA events in an EAGER pass of the same %d steps right after the timed region (%.2f ms/step eager vs %.2f "
                                    "ms/step timed graph replay): events cannot be recorded inside a captured graph; this pass runs on ONE stream (the timed step overlaps teacher / "
                                    "student forward, weight gradients and the discriminator phase on four streams, where an event pair would also time its neighbours)" % (args.steps, ms_eager / args.steps, ms / args.steps)},
    }
    if world == 1 and not args.no_cpu_baseline:
        out["cpu_baseline"] = cpu_baseline_leg()
    if world == 1 and not args.no_context:
        del model
        torch.cuda.empty_cache()
        out["context"] = {"torch_cuda_eager": torch_cuda_eager_context()}
    print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--ref-device", default="cpu", choices=["cpu", "cuda"],
                    help="with --impl reference: cpu = the contract's arm; cuda = the same torch restatement on cuda:0 (context only)")
    ap.add_argument("--ref-tf32", type=int, default=1)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-context", action="store_true", help="skip the torch-on-cuda context measurement (cuDNN eager on the same GPU)")
    ap.add_argument("--conv-table", action="store_true")
    ap.add_argument("--no-graph", action="store_true", help="run every step eagerly instead of replaying CUDA graphs")
    ap.add_argument("--allreduce", default="nccl", choices=["nccl", "nvls"],
                    help="N > 1: nccl = bucketed ncclAllReduce inside the backward pass; nvls = reduction fused into the SGD kernel over NVSwitch multicast")
    ap.add_argument("--allreduce-buckets", type=int, default=4, help="N > 1: ranges of the flat student gradient all-reduced from inside the backward pass (0: one all-reduce after it)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's losses, logits and a parameter sample to DIR/<name>.npy")
    ap.add_argument("--config", type=int, default=3, choices=[3, 4], help="3: BASELINE.json configs[2] (the metric's configuration); 4: the 360x480 batch-16 shape of configs[3]")
    args = ap.parse_args()
    select_config(args.config)
    if args.config == 4:                      # the CPU restatement's discriminator has the reference's fixed head (fails on 46x61 logits)
        args.no_cpu_baseline = True; args.no_context = True
    rank, local_rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29511")
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    if args.warmup < 3:
        args.warmup = 3
    run_ours(args, rank, local_rank, world)


if __name__ == "__main__":
    main()
