"""Cost of the discriminator's self-attention beyond 128 positions.

1. CUDA-event times per call of skd_attn_fwd, skd_attn_tangent_fwd and skd_attn_bwd (first order and joint) at batch 8 for both
   attention shapes of the discriminator, (C, d) = (256, 32) after l3 and (512, 64) after l4, at n = 128 on the default path (the
   whole-tile kernels, except the tangent and joint backward of d = 64, whose tiles do not fit) and forced onto the row-stripe
   kernels (skd_set_attn_tiled(1)), and at n = 144, 256 and 512 (the row-stripe kernels).
2. The distillation step (Pi + Pa + Ho wgan-gp, CUDA graphs) in images/s at 769x769 and 512x1024, batch 8, alternated within one run,
   and the discriminator phase alone (eager, run after the student's step with the device idle) at both crops.

    python -m tools.disc_attention_bench --steps 10 --warmup 4 --rounds 2

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the times do not depend
on the values."""
import argparse
import json

import torch

from tools.espnet_step_bench import _time, card


def attention_times(batch, reps):
    from structure_knowledge_distillation_b200._cabi import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    P = lambda t: None if t is None else t.data_ptr()
    out = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for C, d in ((256, 32), (512, 64)):
        for n, tiled in ((128, 0), (128, 1), (144, 0), (256, 0), (512, 0)):
            B, ldq = batch, 2 * d + C
            r = lambda *s: torch.randn(*s, device="cuda", generator=g)
            qkv, tqkv, x, tx, gy, gty = r(B * n, ldq) * 0.3, r(B * n, ldq) * 0.3, r(B * n, C), r(B * n, C), r(B * n, C), r(B * n, C)
            gamma, gg = torch.tensor([0.3], device="cuda"), torch.zeros(1, device="cuda")
            e = lambda *s: torch.empty(*s, device="cuda")
            attn, dattn, o, y, to, ty, gq, gtq = e(B, n, n), e(B, n, n), e(B * n, C), e(B * n, C), e(B * n, C), e(B * n, C), e(B * n, ldq), e(B * n, ldq)
            L.skd_set_attn_tiled(tiled)
            try:
                ws = e(L.skd_attn_bwd_workspace_floats(B, n, C))
                fwd = lambda: L.skd_attn_fwd(B, n, C, d, P(qkv), ldq, P(x), P(gamma), P(attn), P(o), P(y), None, st)
                tan = lambda: L.skd_attn_tangent_fwd(B, n, C, d, P(qkv), P(tqkv), ldq, P(attn), P(tx), P(gamma), P(dattn), P(to), P(ty), None, st)
                bwd1 = lambda: L.skd_attn_bwd(B, n, C, d, P(qkv), ldq, P(attn), P(o), P(gamma), P(gy), None, None, None, None, P(gq), None,
                                              P(gg), 0, P(ws), st)
                bwd2 = lambda: L.skd_attn_bwd(B, n, C, d, P(qkv), ldq, P(attn), P(o), P(gamma), P(gy), P(tqkv), P(dattn), P(to), P(gty), P(gq),
                                              P(gtq), P(gg), 0, P(ws), st)
                fwd(); tan()
                t = dict(fwd=_time(fwd, reps), tangent=_time(tan, reps), bwd_first_order=_time(bwd1, reps), bwd_joint=_time(bwd2, reps))
            finally:
                L.skd_set_attn_tiled(0)
            key = "C%d_d%d_n%d%s" % (C, d, n, "_forced_row_stripe" if tiled else "")
            out[key] = {k: round(v * 1000.0, 1) for k, v in t.items()}             # microseconds per call
            del qkv, tqkv, x, tx, gy, gty, attn, dattn, o, y, to, ty, gq, gtq, ws
    torch.cuda.empty_cache()
    return out


def _model(batch, h, w, graphs):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", cuda_graph=graphs))
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    return m


def step_rate(batch, h, w, steps, warmup):
    m = _model(batch, h, w, True)
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


def d_phase_ms(batch, h, w, steps, warmup):
    """Eager: the student's forward, backward and update, a synchronise, then the discriminator phase alone between two events."""
    m = _model(batch, h, w, False)
    times = []
    for i in range(warmup + steps):
        m.forward(); m.G_solver.zero_grad(); m.student_backward(); m.G_solver.step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m.discriminator_backward()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(e0.elapsed_time(e1))
    del m
    torch.cuda.empty_cache()
    return sum(times) / len(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--skip-steps", action="store_true", help="kernel times only")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, attention_us_per_call=attention_times(a.batch, a.reps))
    if not a.skip_steps:
        res.update(losses="Pi+Pa+Ho wgan-gp", cuda_graph=True, step={"769x769": [], "512x1024": []}, d_phase_eager_ms={"769x769": [], "512x1024": []})
        for _ in range(a.rounds):
            for name, h, w in (("769x769", 769, 769), ("512x1024", 512, 1024)):
                ips, ms = step_rate(a.batch, h, w, a.steps, a.warmup)
                res["step"][name].append(dict(images_per_s=round(ips, 2), ms_per_step=round(ms, 2)))
                res["d_phase_eager_ms"][name].append(round(d_phase_ms(a.batch, h, w, a.steps, 2), 2))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
