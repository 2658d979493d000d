"""Time the teacher's short-K 1x1 convolutions (PSPNet-101 bottleneck shapes at the benchmark's batch 8 @512x1024) in isolation.

Each shape runs through ops.conv2d_fwd as the frozen teacher calls it (folded BN as scale / shift, residual added in place, ReLU),
timed with CUDA events over --iters launches after --warmup.  Printed per shape: ms per launch, TFLOP/s, and GB/s of algorithmic
bytes (input, weights, residual read once, output written once).  For the ceiling this card reaches, the same process times a torch
device-to-device copy moving the same number of bytes (half read, half written).

    python -m tools.conv_epilogue_bench [--iters 500] [--warmup 10]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# name, N, Cin, H, W, Cout, residual
SHAPES = [
    ("layer3 conv3 1x1 256->1024 +BN +res +ReLU", 8, 256, 65, 129, 1024, True),
    ("layer4 conv3 1x1 512->2048 +BN +res +ReLU", 8, 512, 65, 129, 2048, True),
    ("layer1 conv3 1x1 64->256 +BN +res +ReLU", 8, 64, 129, 257, 256, True),
    ("layer3 conv1 1x1 1024->256 +BN +ReLU", 8, 1024, 65, 129, 256, False),
]


def card(index):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"nvidia-smi": "unavailable"}


def time_ms(fn, iters, warmup, index):
    """-> (ms per call, median SM MHz sampled from the warm-up to the end of the timed calls)"""
    import torch
    from bench import ClockSampler
    clocks = ClockSampler(index)
    clocks.start()
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters, clocks.stop()["sm_mhz"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert args.iters >= 50, "time at least 50 launches"
    import torch
    from structure_knowledge_distillation_b200 import ops
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    index = torch.cuda.current_device()
    print("card:", torch.cuda.get_device_name(dev), card(index))
    rows = []
    for name, N, Cin, H, W, Cout, with_res in SHAPES:
        x = ops.to_nhwc(torch.randn(N, Cin, H, W, device=dev, generator=g))
        w = ops.weight_ohwi(torch.randn(Cout, Cin, 1, 1, device=dev, generator=g) / Cin ** 0.5)
        sc = torch.rand(Cout, device=dev, generator=g) + 0.5
        sh = torch.randn(Cout, device=dev, generator=g) * 0.1
        out = ops.to_nhwc(torch.randn(N, Cout, H, W, device=dev, generator=g))
        res = out if with_res else None                  # in place, as Bottleneck.frozen adds its identity path

        def conv():
            ops.conv2d_fwd(x, w, 1, 0, 1, scale=sc, shift=sh, residual=res, act="relu", out=out)

        P = N * H * W
        flop = 2.0 * P * Cin * Cout
        nbytes = 4 * (P * Cin + Cout * Cin + P * Cout * (2 if with_res else 1))
        ms, mhz = time_ms(conv, args.iters, args.warmup, index)
        src = torch.empty(nbytes // 8, device=dev)
        dst = torch.empty_like(src)
        ms_copy, mhz_copy = time_ms(lambda: dst.copy_(src), args.iters, args.warmup, index)
        del src, dst
        rows.append((name, ms, flop / ms / 1e9, nbytes / ms / 1e6, nbytes / ms_copy / 1e6, mhz, mhz_copy))
    print("%-44s %8s %8s %7s %9s %8s %9s %9s" % ("shape (batch 8)", "ms", "TFLOP/s", "GB/s", "copy GB/s", "of copy", "SM MHz", "copy MHz"))
    for name, ms, tf, gbs, cgbs, mhz, cmhz in rows:
        print("%-44s %8.3f %8.1f %7.0f %9.0f %7.0f%% %9s %9s" % (name, ms, tf, gbs, cgbs, 100 * gbs / cgbs, mhz, cmhz))


if __name__ == "__main__":
    main()
