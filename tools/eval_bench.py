"""Throughput of the evaluation path on one GPU: evaluate_main (whole image, 1024x2048) on the student with the default single
scale and with the six-scale + flip setting, the zoom and paired-accumulate kernels alone, and whether writing PNGs (png_dir)
changes the image rate.  Prints one JSON line (and writes it to --out when given) with the card's name and power limit.

    python -m tools.eval_bench [--images 6] [--repeats 3] [--out result.json]

Work per image, for context (arithmetic, not a timing): the student forward is ~1.0 TFLOP at 1024x2048 (4 x 251.7 GFLOP at
512x1024, SURVEY.md), and scales s with flip cost 2 * sum(s^2) forwards: 17.375 for (0.5 .. 1.75) + flip, ~17.4 TFLOP.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIX = (0.5, 0.75, 1.0, 1.25, 1.5, 1.75)
FWD_TFLOP_1024x2048 = 4 * 0.2517


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the rate is still worth printing; the card is then unknown
        q = "unknown (%s)" % e
    return q


def batches(n, H=1024, W=2048, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        image = (torch.randn(1, 3, H, W, generator=g) * 50).cuda()
        label = torch.randint(0, 19, (1, H, W), generator=g).cuda()
        out.append((image, label, [np.array([H, W, 3])], ["bench%d" % i]))
    return out


def rate(net, data, scales, flip, png_dir=None):
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    torch.cuda.synchronize()
    t = time.perf_counter()
    evaluate_main(net, data, 0, "512,512", 19, whole=True, scales=scales, flip=flip, png_dir=png_dir)
    torch.cuda.synchronize()
    return len(data) / (time.perf_counter() - t)


def kernel_ms(fn, launches):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=6)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "eval_bench measures the GPU; there is no CPU number"
    from structure_knowledge_distillation_b200._cabi import lib
    from structure_knowledge_distillation_b200.networks.evaluate import zoom_image
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Res_pspnet
    torch.manual_seed(0)
    net = Res_pspnet(BasicBlock, [2, 2, 2, 2], 19).cuda().eval()
    data = batches(args.images)
    res = dict(card=card(), images=args.images, repeats=args.repeats)
    # warm every shape first (each scale's forward, flip batch 2, the PNG writer)
    with tempfile.TemporaryDirectory() as tmp:
        rate(net, data[:1], (1.0,), False)
        rate(net, data[:1], SIX, True)
        rate(net, data[:1], (1.0,), False, png_dir=tmp)
        single, multi, single_png = [], [], []
        for _ in range(args.repeats):                      # alternate the settings so drift hits them alike
            single.append(rate(net, data, (1.0,), False))
            single_png.append(rate(net, data, (1.0,), False, png_dir=tmp))
            multi.append(rate(net, data[:max(1, args.images // 3)], SIX, True))
    res["single_scale_images_per_s"] = [round(r, 2) for r in single]
    res["single_scale_png_images_per_s"] = [round(r, 2) for r in single_png]
    res["six_scale_flip_images_per_s"] = [round(r, 3) for r in multi]
    work = 2 * sum(s * s for s in SIX)
    res["six_scale_flip_forward_work_x"] = work
    res["six_scale_flip_tflop_per_image_arith"] = round(work * FWD_TFLOP_1024x2048, 2)
    # kernels alone: zoom with flip at 1.75 (the largest output), paired accumulate of 19-class 1/8 logits into 1024x2048
    image = data[0][0]
    res["zoom_flip_ms"] = {str(s): round(kernel_ms(lambda: zoom_image(image, s, True), args.launches), 4) for s in (0.5, 1.0, 1.75)}
    logits = torch.randn(2, 128, 256, 20, device="cuda").permute(0, 3, 1, 2)[:, :19]
    full = torch.zeros(1024, 2048, 19, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def acc(paired):
        return lambda: lib().skd_eval_upsample_accumulate_ms(19, 128, 256, logits.data_ptr(), 128 * 256 * 20, 1, 20, 1024, 2048, 1024, 2048,
                                                             full.data_ptr(), 2048, 1.0 / 6, paired, st)
    res["accumulate_paired_ms"] = round(kernel_ms(acc(1), args.launches), 4)
    res["accumulate_single_ms"] = round(kernel_ms(acc(0), args.launches), 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
