"""Time the weight-gradient convolutions of the benchmark step (batch 8, at 65x129 unless noted) with and without Cout tile pairs,
in isolation.

Each shape runs through ops.conv2d_wgrad (the wgmma kernel plus its split-K reduce), timed with CUDA events over --iters launches
after --warmup.  The pairing modes are selected with skd_set_wgrad_pairing (0 = single units only, 1 = automatic, 2 = every legal
pair) and alternated --rounds times per shape, so all see the same clock and the same neighbours.  Printed per shape and mode: the
pair units of the launch, the median ms per launch over the rounds, the range, TFLOP/s of the median, and the median SM clock;
then the gain of mode 1 over mode 0 and, for shapes with pairs, the time r of a pair in single-unit times implied by modes 0 and 2,
each a static stride over 132 CTAs.  Cout >= 256 (Cout tile pairs, a pair launch then a single launch): mode 0 takes
ceil(units / 132), mode 2 ceil(pairs / 132) r + ceil(singles / 132).  Cout <= 64 (one unit per warpgroup, one launch of
units - pairs items): mode 2 takes ceil(items / 132) + (r - 1) ceil(pairs / 132).

    python -m tools.conv_wgrad_bench [--iters 50] [--warmup 10] [--rounds 3]
"""
import argparse
import ctypes
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.conv_epilogue_bench import card, time_ms  # noqa: E402

# name, Cin, Cout, k, stride, pad, dil[, H, W]: the step's weight gradients (tests/test_conv_exact_gpu.py inventory); the Cout >= 256
# launches with 128-channel Cin tiles and the Cout <= 64 ones with Cin <= 64 can pair, the others are single-unit launches.
SHAPES = [
    ("layer4 3x3 d4 512->512", 512, 512, 3, 1, 4, 4),
    ("layer4 3x3 d4 256->512", 256, 512, 3, 1, 4, 4),
    ("layer3 3x3 d2 256->256", 256, 256, 3, 1, 2, 2),
    ("layer3 3x3 d2 128->256", 128, 256, 3, 1, 2, 2),
    ("layer4 downsample 1x1 256->512", 256, 512, 1, 1, 0, 1),
    ("layer3 downsample 1x1 128->256", 128, 256, 1, 1, 0, 1),
    ("head 3x3 1024->128", 1024, 128, 3, 1, 1, 1),
    ("layer2 3x3 128->128", 128, 128, 3, 1, 1, 1),
    ("layer1 3x3 64->64 at 129x257", 64, 64, 3, 1, 1, 1, 129, 257),
    ("stem conv2 3x3 64->64 at 256x512", 64, 64, 3, 1, 1, 1, 256, 512),
]
N, H0, W0 = 8, 65, 129
MODES = (0, 1, 2)
SMS = 132


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert args.iters >= 50, "time at least 50 launches"
    import torch
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    index = torch.cuda.current_device()
    print("card:", torch.cuda.get_device_name(dev), card(index))
    L = lib()
    rows = []
    try:
        for name, Cin, Cout, k, s, pad, dil, *hw in SHAPES:
            H, W = hw or (H0, W0)
            OH, OW = (H + 2 * pad - dil * (k - 1) - 1) // s + 1, (W + 2 * pad - dil * (k - 1) - 1) // s + 1
            x = ops.to_nhwc(torch.randn(N, Cin, H, W, device=dev, generator=g))
            dy = ops.to_nhwc(torch.randn(N, Cout, OH, OW, device=dev, generator=g))

            def conv():
                ops.conv2d_wgrad(x, dy, (k, k), s, pad, dil)
            flop = 2.0 * N * OH * OW * Cin * Cout * k * k
            res = {m: ([], [], None, None) for m in MODES}
            for _ in range(args.rounds):
                for m in MODES:
                    L.skd_set_wgrad_pairing(m)
                    ms, mhz = time_ms(conv, args.iters, args.warmup, index)
                    plan, pairs = (ctypes.c_int * 3)(), (ctypes.c_int * 1)()
                    L.skd_conv_wgrad_last_plan(plan)
                    L.skd_conv_wgrad_last_pairs(pairs)
                    res[m][0].append(ms)
                    res[m][1].append(mhz)
                    res[m] = (res[m][0], res[m][1], list(plan), pairs[0])
            rows.append((name, Cin, Cout, k, flop, res))
    finally:
        L.skd_set_wgrad_pairing(1)
    print("%-36s %4s %5s %8s %17s %8s %8s" % ("shape (batch 8)", "mode", "pairs", "ms", "range", "TFLOP/s", "SM MHz"))
    for name, Cin, Cout, k, flop, res in rows:
        for m in MODES:
            ms_l, mhz_l, plan, pairs = res[m]
            med = statistics.median(ms_l)
            mhz = [v for v in mhz_l if v is not None]
            print("%-36s %4d %5d %8.3f %8.3f-%8.3f %8.1f %8s" % (name, m, pairs, med, min(ms_l), max(ms_l), flop / med / 1e9,
                                                                 statistics.median(mhz) if mhz else "n/a"))
        t0, t1 = statistics.median(res[0][0]), statistics.median(res[1][0])
        line = "%-36s gain of mode 1 over 0: %+.1f%%" % ("", 100.0 * (t0 / t1 - 1.0))
        plan, pairs2 = res[2][2], res[2][3]
        if pairs2:
            bn, splits = plan[0], plan[2]
            units = _units(Cin, Cout, k, bn, splits)
            t2 = statistics.median(res[2][0])
            u = t0 / math.ceil(units / SMS)
            if Cout <= 64:
                items = units - pairs2
                grid = min(items, SMS)
                r = 1.0 + (t2 / u - math.ceil(items / grid)) / math.ceil(pairs2 / grid)
            else:
                r = (t2 / u - math.ceil((units - 2 * pairs2) / SMS)) / math.ceil(pairs2 / SMS)
            line += ", pair / single unit time implied by modes 0 and 2: %.2f" % r
        print(line)


def _units(Cin, Cout, k, bn, splits):
    return math.ceil(Cout / 128) * math.ceil(Cin / bn) * k * k * splits


if __name__ == "__main__":
    main()
