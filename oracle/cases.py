"""Seeded test cases shared by oracle/make_golden.py (which runs the REAL reference on them) and the tests
(which run oracle/port.py and the CUDA path on them).  TEST INFRASTRUCTURE ONLY.

Model weights are never stored: they are re-created from a seed by constructing the *port* modules (state-dict
names identical to the reference's, so the same tensors are loaded into the reference for golden generation).
"""
import torch

from . import port


def seeded(seed):
    return torch.Generator().manual_seed(seed)


def build_models(seed=0, with_D=True, classes=19):
    """Teacher / student / D with default torch init under a fixed seed, BN stats perturbed (SURVEY §8d)."""
    torch.manual_seed(seed)
    student = port.PSPNet("resnet18", classes)
    teacher = port.PSPNet("resnet101", classes)
    D = port.Discriminator(1, classes, 64) if with_D else None
    port.perturb_bn_stats(teacher, seed + 1)
    port.perturb_bn_stats(student, seed + 2)
    return teacher, student, D


def dropout_masks(student, batch, seed):
    g = seeded(seed)
    masks = []
    for d, c in zip(student.dropouts(), (student.pspmodule.bottleneck[0].out_channels, student.dsn[0].out_channels)):
        masks.append((torch.rand(batch, c, generator=g) >= d.p).float())
    return masks


def criterion_inputs(n, c_s, c_t, classes, h, w, seed):
    """Random 7-lists shaped like Res_pspnet outputs (only indices 0,1,2 are read by the criteria)."""
    g = seeded(seed)
    def r(*s):
        return torch.randn(*s, generator=g)
    S = [r(n, classes, h, w) * 2, r(n, classes, h, w) * 2, r(n, c_s, h, w), None, None, None, None]
    T = [r(n, classes, h, w) * 2, r(n, classes, h, w) * 2, r(n, c_t, h, w), None, None, None, None]
    return S, T


CRITERION_CASES = [
    # name, n, c_s, c_t, h, w, pool_scale, label_hw
    ("tiny", 1, 8, 16, 9, 9, 0.5, (64, 64)),
    ("ragged", 2, 16, 24, 13, 17, 0.25, (97, 131)),
    ("nodes81", 2, 32, 64, 33, 65, 0.125, (130, 258)),
    ("unpooled", 1, 16, 32, 9, 12, 1.0 / 9, (30, 41)),
]

STEP_CASES = {
    # name: (batch, H, W, cfg kwargs)
    "cfg1_pi_64": dict(batch=1, h=64, w=64, cfg=dict(pi=True, pa=False, ho=False)),
    "pi_pa_96x128": dict(batch=2, h=96, w=128, cfg=dict(pi=True, pa=True, ho=False, pool_scale=0.5)),
    "pi_pa_ho_hinge_512": dict(batch=1, h=512, w=512, cfg=dict(pi=True, pa=True, ho=True, adv_type="hinge")),
    "pi_pa_ho_wgangp_512": dict(batch=1, h=512, w=512, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
}

# BASELINE.json configs[2] at full size (batch 8 @ 512x1024, Pi+Pa+Ho, wgan-gp): generated once by
# `python -m oracle.make_golden --full` (several minutes of CPU), checked on the H100 by tests/test_step_gpu.py.
FULL_CASES = {
    "baseline_cfg3_b8_512x1024": dict(batch=8, h=512, w=1024, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
}


# BASELINE.json configs[3] shape (360x480 CamVid crops -> 46x61 logits), ResNet18 student (the reference ships no ESPNet source).
# Pi+Pa only: the reference's own discriminator cannot run on 46x61 logits (sagan_models.py:131-136,163); our size-aware head is
# checked against oracle/port.py with the same head in tests/test_discriminator_gpu.py.  `python -m oracle.make_golden --cfg4`.
CFG4_CASES = {
    "cfg4_pi_pa_360x480_b2": dict(batch=2, h=360, w=480, cfg=dict(pi=True, pa=True, ho=False, pool_scale=0.5)),
}


def sample_large(t, k=8192, limit=20000):
    """A stored reference tensor above `limit` elements is kept as a fixed sample of flat positions, {"idx", "val"}, so that
    every fixture stays below 1 MB; the positions depend only on the element count."""
    if t.numel() <= limit:
        return t
    g = torch.Generator().manual_seed(t.numel())
    idx = torch.randperm(t.numel(), generator=g)[:k].sort().values
    return {"idx": idx.to(torch.int32), "val": t.flatten()[idx].clone()}


def at_stored(t, stored):
    """(values of `t`, reference values) at the positions a stored reference tensor keeps (all of them when it is not sampled)."""
    if isinstance(stored, dict):
        return t.flatten()[stored["idx"].long().to(t.device)], stored["val"]
    return t, stored


def stored_sum(a, b):
    """Sum of two stored reference tensors of the same shape (sampled at the same positions)."""
    if isinstance(a, dict):
        return {"idx": a["idx"], "val": a["val"] + b["val"]}
    return a + b


def grad_digest(named_params, k=16):
    """Small fingerprint of each gradient: l2 norm, sum, and k strided samples."""
    out = {}
    for name, p in named_params:
        if p.grad is None:
            continue
        g = p.grad.detach().flatten().double()
        idx = torch.linspace(0, g.numel() - 1, min(k, g.numel())).long()
        out[name] = dict(norm=float(g.norm()), sum=float(g.sum()), samples=g[idx].float().clone(), idx=idx)
    return out
