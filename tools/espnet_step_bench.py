"""Cost of the ESPNet students: the config-4 distillation step (batch 16 at 360x480, Pi+Pa+Ho wgan-gp, CUDA graphs) with the
ResNet18-PSP, ESPNet-C and full ESPNet students, alternated within one run, and CUDA-event times of the ESPNet kernels at that shape
(the full ESPNet's transposed convolutions and the adjoint of its logits' resize onto the teacher's grid included).

    python -m tools.espnet_step_bench --steps 20 --warmup 5 --rounds 2

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the rates do not depend
on the values."""
import argparse
import json
import subprocess

import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def step_rate(student, batch, steps, warmup):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", student=student, cuda_graph=True))
    images, labels = port.synthetic_batch(batch, 360, 480, seed=1)
    m.set_input((images, labels, None, None))
    for _ in range(warmup):
        m.optimize_parameters()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.optimize_parameters()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del m
    torch.cuda.empty_cache()
    return batch * 1000.0 / ms, ms


def _time(fn, reps=200):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_times(batch):
    """ms per call at the config-4 shapes: b1 (19 channels at 180x240), the level-3 ESP combine (128 channels at 45x60), the input
    projections and the teacher resample (46x61 -> 45x60 of the logits and the 512-channel feature)."""
    from structure_knowledge_distillation_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    dev = "cuda"
    out = {}
    x = ops.empty_nhwc(batch, 19, 180, 240, dev, pitch=20); x.normal_(generator=g)
    c = 19
    w, b, a = torch.ones(c, device=dev), torch.zeros(c, device=dev), torch.full((c,), 0.25, device=dev)
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    st = ops.bnprelu_stats(x, 0.1, rm, rv, None)
    dy = ops.empty_nhwc(batch, 20, 180, 240, dev); dy.normal_(generator=g)
    out["bnprelu_stats_b1"] = _time(lambda: ops.bnprelu_stats(x, 0.1, rm, rv, None))
    out["bnprelu_apply_b1"] = _time(lambda: ops.bnprelu_apply(x, st[0], st[1], w, b, a, 1e-3, out_channels=20))
    red = ops.bnprelu_bwd_reduce(x, dy, st[0], st[1], w, b, a, 1e-3)
    out["bnprelu_bwd_reduce_b1"] = _time(lambda: ops.bnprelu_bwd_reduce(x, dy, st[0], st[1], w, b, a, 1e-3))
    out["bnprelu_bwd_dx_b1"] = _time(lambda: ops.bnprelu_bwd_dx(x, dy, st[0], st[1], w, b, a, 1e-3, True, red[3], dx_channels=20))
    n, n1, C = 25, 28, 128
    br = [ops.empty_nhwc(batch, n1, 45, 60, dev, pitch=28)] + [ops.empty_nhwc(batch, n, 45, 60, dev, pitch=28) for _ in range(4)]
    for t in br:
        t.normal_(generator=g)
    res = ops.empty_nhwc(batch, C, 45, 60, dev); res.normal_(generator=g)
    comb = ops.empty_nhwc(batch, C, 45, 60, dev)
    w, b, a = torch.ones(C, device=dev), torch.zeros(C, device=dev), torch.full((C,), 0.25, device=dev)
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    st = ops.esp_combine(br, res, comb, 0.1, rm, rv, None)
    dyc = ops.empty_nhwc(batch, C, 45, 60, dev); dyc.normal_(generator=g)
    red = ops.bnprelu_bwd_reduce(comb, dyc, st[0], st[1], w, b, a, 1e-3)
    out["esp_combine_stats_l3"] = _time(lambda: ops.esp_combine(br, res, comb, 0.1, rm, rv, None))
    out["esp_bwd_dx_l3"] = _time(lambda: ops.esp_bwd_dx(comb, dyc, st[0], st[1], w, b, a, 1e-3, True, red[3], n1, n, True))
    img = ops.empty_nhwc(batch, 4, 360, 480, dev); img.normal_(generator=g)
    cat1 = ops.empty_nhwc(batch, 20, 180, 240, dev)
    cat2 = ops.empty_nhwc(batch, 132, 90, 120, dev)
    out["input_projection_1"] = _time(lambda: ops.avgpool3x3s2(img[:, :3], cat1[:, 16:19]))
    out["input_projection_2"] = _time(lambda: ops.avgpool3x3s2(cat1[:, 16:19], cat2[:, 128:131]))
    lt = ops.empty_nhwc(batch, 19, 46, 61, dev, pitch=20); lt.normal_(generator=g)
    ft = ops.empty_nhwc(batch, 512, 46, 61, dev); ft.normal_(generator=g)
    out["resample_teacher_logits"] = _time(lambda: ops.resample_nhwc(lt, 45, 60), 50)
    out["resample_teacher_feat"] = _time(lambda: ops.resample_nhwc(ft, 45, 60), 50)
    # the full ESPNet: up_l3 (1/8 -> 1/4), up_l2 (1/4 -> 1/2) and classifier (1/2 -> 1/1) forward, data and weight gradients
    from structure_knowledge_distillation_b200 import functions as Fn
    wt = torch.randn(19, 19, 2, 2, device=dev, generator=g)
    for name, (h, w) in (("up_l3", (45, 60)), ("up_l2", (90, 120)), ("classifier", (180, 240))):
        xt = ops.empty_nhwc(batch, 20, h, w, dev); xt.normal_(generator=g)
        dyt = ops.empty_nhwc(batch, 20, 2 * h, 2 * w, dev); dyt.normal_(generator=g)
        wd = torch.zeros(20, 2, 2, 20, device=dev); wd[:19, :, :, :19] = wt.permute(0, 2, 3, 1)
        wr = torch.zeros(2, 2, 20, 20, device=dev); wr[:, :, :19, :19] = wt.permute(2, 3, 1, 0)
        wr = wr.reshape(2, 40, 1, 1, 20)
        out["convT_fwd_" + name] = _time(lambda: ops.conv_transpose2x2_fwd(xt, wr), 50)
        out["convT_dgrad_" + name] = _time(lambda: ops.conv2d_fwd(dyt, wd, 2, 0, 1), 50)
        out["convT_wgrad_" + name] = _time(lambda: ops.conv2d_wgrad(dyt, xt, (2, 2), 2, 0, 1), 50)
    ls = ops.empty_nhwc(batch, 19, 360, 480, dev, pitch=20); ls.normal_(generator=g)
    out["resize_student_logits_to_teacher"] = _time(lambda: Fn.ResampleBilinear.apply(ls, 46, 61), 50)
    dd = torch.randn(batch, 19, 46, 61, device=dev, generator=g)
    out["resize_adjoint"] = _time(lambda: ops.resample_adjoint_nhwc(dd, 360, 480), 50)
    return {k: round(v, 4) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, shape="360x480", losses="Pi+Pa+Ho wgan-gp", cuda_graph=True, resnet18=[], espnet_c=[],
               espnet=[])
    for _ in range(a.rounds):
        for student in ("resnet18", "espnet_c", "espnet"):
            ips, ms = step_rate(student, a.batch, a.steps, a.warmup)
            res[student].append(dict(images_per_s=round(ips, 2), ms_per_step=round(ms, 2)))
    res["kernels_ms"] = kernel_times(a.batch)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
