"""Time the convolutions of the benchmark step (batch 8, at 65x129 unless noted) on 128-row and on 256-row wgmma tiles, in isolation.

Each shape runs through ops.conv2d_fwd with its folded BN as scale / shift and ReLU (or ops.conv2d_dgrad for the data gradient), timed
with CUDA events over --iters launches after --warmup.  The two tile paths are selected with skd_set_conv_tile_m (1 = 128 rows,
2 = 256 rows) and alternated --rounds times per shape, so both see the same clock and the same neighbours.  Printed per shape and
path: the median ms per launch over the rounds, the range, TFLOP/s of the median, and the median SM clock.

    python -m tools.conv_tile_bench [--iters 50] [--warmup 10] [--rounds 3]
"""
import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.conv_epilogue_bench import card, time_ms  # noqa: E402

# name, kind, Cin, Cout, k, pad, dil[, H, W]  (batch 8, 65x129 input unless given; fwd: folded BN + ReLU; dgrad: the stride-1 data
# gradient, no epilogue).  The long-K shapes set the rate of the 256-row path; the short-K ones (K = 2 .. 72 steps) and the lone N
# tile of the 3x3 1024->128 are the launches the tile selection in conv_fwd_impl decides on.
SHAPES = [
    ("PSP bottleneck 3x3 4096->512", "fwd", 4096, 512, 3, 1, 1),
    ("DSN head 3x3 1024->512", "fwd", 1024, 512, 3, 1, 1),
    ("layer3 3x3 d2 256->256", "fwd", 256, 256, 3, 2, 2),
    ("layer4 3x3 d4 512->512", "fwd", 512, 512, 3, 4, 4),
    ("layer4 1x1 2048->512", "fwd", 2048, 512, 1, 0, 1),
    ("layer4 downsample 1x1 1024->2048", "fwd", 1024, 2048, 1, 0, 1),
    ("layer3 1x1 1024->256", "fwd", 1024, 256, 1, 0, 1),
    ("1x1 1024->512", "fwd", 1024, 512, 1, 0, 1),
    ("layer3 downsample 1x1 512->1024", "fwd", 512, 1024, 1, 0, 1),
    ("1x1 512->128", "fwd", 512, 128, 1, 0, 1),
    ("layer1 downsample 1x1 64->256 at 129x257", "fwd", 64, 256, 1, 0, 1, 129, 257),
    ("head 3x3 1024->128", "fwd", 1024, 128, 3, 1, 1),
    ("stem 3x3 64->128 at 256x512", "fwd", 64, 128, 3, 1, 1, 256, 512),
    ("dgrad layer4 3x3 d4 512->512", "dgrad", 512, 512, 3, 4, 4),
    ("dgrad layer4 3x3 d4 256->512", "dgrad", 256, 512, 3, 4, 4),
    ("dgrad layer3 3x3 d2 256->256", "dgrad", 256, 256, 3, 2, 2),
    ("dgrad layer3 3x3 d2 128->256", "dgrad", 128, 256, 3, 2, 2),
]
N, H0, W0 = 8, 65, 129
PATHS = ((1, "128"), (2, "256"))


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
        for name, kind, Cin, Cout, k, pad, dil, *hw in SHAPES:
            H, W = hw or (H0, W0)
            w = ops.weight_ohwi(torch.randn(Cout, Cin, k, k, device=dev, generator=g) / (Cin * k * k) ** 0.5)
            if kind == "fwd":
                x = ops.to_nhwc(torch.randn(N, Cin, H, W, device=dev, generator=g))
                sc = torch.rand(Cout, device=dev, generator=g) + 0.5
                sh = torch.randn(Cout, device=dev, generator=g) * 0.1
                out = ops.empty_nhwc(N, Cout, H, W, dev)

                def conv():
                    ops.conv2d_fwd(x, w, 1, pad, dil, scale=sc, shift=sh, act="relu", out=out)
            else:
                dy = ops.to_nhwc(torch.randn(N, Cout, H, W, device=dev, generator=g))

                def conv():
                    ops.conv2d_dgrad(dy, w, (N, Cin, H, W), 1, pad, dil)
            flop = 2.0 * N * H * W * Cin * Cout * k * k
            res = {p: ([], []) for _, p in PATHS}
            for _ in range(args.rounds):
                for mode, p in PATHS:
                    L.skd_set_conv_tile_m(mode)
                    ms, mhz = time_ms(conv, args.iters, args.warmup, index)
                    res[p][0].append(ms)
                    res[p][1].append(mhz)
            rows.append((name, flop, res))
    finally:
        L.skd_set_conv_tile_m(0)
    print("%-42s %5s %8s %17s %8s %8s" % ("shape (batch 8)", "tile", "ms", "range", "TFLOP/s", "SM MHz"))
    for name, flop, res in rows:
        for _, p in PATHS:
            ms_l, mhz_l = res[p]
            med = statistics.median(ms_l)
            mhz = [m for m in mhz_l if m is not None]
            print("%-42s %5s %8.3f %8.3f-%8.3f %8.1f %8s" % (name, p, med, min(ms_l), max(ms_l), flop / med / 1e9,
                                                            statistics.median(mhz) if mhz else "n/a"))
        print("%-42s %5s %7.1f%%" % ("", "gain", 100.0 * (statistics.median(res["128"][0]) / statistics.median(res["256"][0]) - 1.0)))


if __name__ == "__main__":
    main()
