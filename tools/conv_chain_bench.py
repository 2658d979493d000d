"""Time the frozen teacher's bottleneck 1x1 pairs (block i's conv3 with folded BN + residual + ReLU, block i+1's conv1 with folded
BN + ReLU) at the benchmark's batch 8, as one chained launch (ops.conv1x1_chain) and as the two launches it replaces, in isolation.

Alternated --rounds times per shape with CUDA events over --iters calls after --warmup.  Beside them: a device-to-device copy that
moves the chain's HBM bytes (x3, residual and y3 once each, y1 once), the rate those bytes allow.  Printed per shape: median ms per
call, the range over rounds, TFLOP/s of both convolutions, the copy's ms and the median SM clock; the card's name, power limit and
maximum SM clock come first.

    python -m tools.conv_chain_bench [--iters 50] [--warmup 10] [--rounds 3]
"""
import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.conv_epilogue_bench import card, time_ms  # noqa: E402

# name, N, planes, H, W: conv3 planes -> 4 * planes, then conv1 4 * planes -> planes
PAIRS = [
    ("layer1 64->256->64 @129x257", 8, 64, 129, 257),
    ("layer2 128->512->128 @65x129", 8, 128, 65, 129),
    ("layer3 256->1024->256 @65x129", 8, 256, 65, 129),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
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
    for name, N, planes, H, W in PAIRS:
        c3 = 4 * planes
        x3 = ops.to_nhwc(torch.relu(torch.randn(N, planes, H, W, device=dev, generator=g)))
        res = ops.to_nhwc(torch.randn(N, c3, H, W, device=dev, generator=g))
        w3 = ops.weight_ohwi(torch.randn(c3, planes, 1, 1, device=dev, generator=g) / planes ** 0.5)
        w1 = ops.weight_ohwi(torch.randn(planes, c3, 1, 1, device=dev, generator=g) / c3 ** 0.5)
        sc3, sh3 = torch.rand(c3, device=dev, generator=g) + 0.5, torch.randn(c3, device=dev, generator=g) * 0.1
        sc1, sh1 = torch.rand(planes, device=dev, generator=g) + 0.5, torch.randn(planes, device=dev, generator=g) * 0.1
        y3 = ops.empty_nhwc(N, c3, H, W, dev)
        y1 = ops.empty_nhwc(N, planes, H, W, dev)
        P = N * H * W
        hbm_bytes = 4 * P * (planes + 2 * c3 + planes)
        src = torch.empty(hbm_bytes // 8, device=dev)
        dst = torch.empty_like(src)

        def chain():
            ops.conv1x1_chain(x3, w3, sc3, sh3, res, w1, sc1, sh1, out3=y3)

        def two():
            ops.conv2d_fwd(x3, w3, 1, 0, 1, scale=sc3, shift=sh3, residual=res, act="relu", out=y3)
            ops.conv2d_fwd(y3, w1, 1, 0, 1, scale=sc1, shift=sh1, act="relu", out=y1)

        def copy():
            dst.copy_(src)

        res_t = {k: ([], []) for k in ("two launches", "chain", "copy")}
        for _ in range(args.rounds):
            for k, fn in (("two launches", two), ("chain", chain), ("copy", copy)):
                ms, mhz = time_ms(fn, args.iters, args.warmup, index)
                res_t[k][0].append(ms)
                res_t[k][1].append(mhz)
        rows.append((name, 2.0 * P * c3 * 2 * planes, hbm_bytes, res_t))
    print("%-32s %-13s %8s %17s %8s %8s %8s" % ("pair (batch 8)", "path", "ms", "range", "TFLOP/s", "GB/s", "SM MHz"))
    for name, flop, nbytes, res_t in rows:
        for k, (ms_l, mhz_l) in res_t.items():
            med = statistics.median(ms_l)
            mhz = [m for m in mhz_l if m is not None]
            print("%-32s %-13s %8.3f %8.3f-%8.3f %8s %8.0f %8s" % (
                name, k, med, min(ms_l), max(ms_l), "%.1f" % (flop / med / 1e9) if k != "copy" else "", nbytes / med / 1e6,
                statistics.median(mhz) if mhz else "n/a"))
        print("%-32s %-13s %7.1f%%" % ("", "chain gain", 100.0 * (statistics.median(res_t["two launches"][0]) /
                                                                 statistics.median(res_t["chain"][0]) - 1.0)))


if __name__ == "__main__":
    main()
