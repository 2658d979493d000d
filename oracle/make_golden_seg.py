"""TEST INFRASTRUCTURE -- generates tests/golden/seg_steps.pt.gz: plain segmentation training steps (no teacher, no discriminator) of the
UNMODIFIED reference on the CPU, and pins oracle/port.py's training-mode PSPNet against them on the spot.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_seg

Each case builds `Res_pspnet` in train mode (networks/pspnet_combine.py) with seeded weights, the two head dropouts replaced by the
injected masks of cases.dropout_masks(seed=2), and `optim.SGD` constructed as networks/kd_model.py:74 constructs G_solver, then runs
two steps of: zero_grad -> forward -> CriterionDSN (or CriterionOhemDSN) -> backward -> SGD step, at a constant learning rate.
Recorded per step: the loss, the logits, the digest of every gradient (l2 norm, sum, 16 strided samples) and the parameters
at the same positions after the SGD step.

Cases (`CASES`): PSPNet-ResNet101 at 19 and 21 classes with CriterionDSN, at 19 classes with CriterionOhemDSN (a threshold below every
probability, so the kept set is the `OHEM_KEEP` hardest pixels and not all of them), and the ResNet18-PSP student alone -- the
reference's "baseline" row, trained without distillation.  All batch 2 at 96 x 128.
"""
import contextlib
import gzip
import io
import os
import re
import time

import torch

from . import cases, port, refshim
from .make_golden import _cpu_cuda_patch, _rel

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "seg_steps.pt.gz")

BATCH, H, W = 2, 96, 128
STEPS = 2
LR, MOMENTUM, WEIGHT_DECAY = 1e-2, 0.9, 5e-4
OHEM_THRES, OHEM_KEEP = 0.01, 5000
NET_SEED = 0
CASES = {
    # name: (network, classes, ohem)
    "r101_c19": ("resnet101", 19, False),
    "r101_c21": ("resnet101", 21, False),
    "r101_c19_ohem": ("resnet101", 19, True),
    "r18_c19": ("resnet18", 19, False),
}


def build_net(arch, classes):
    """The port network of a case, with its seeded weights and perturbed BN statistics / affine parameters."""
    torch.manual_seed(NET_SEED)
    net = port.PSPNet(arch, classes)
    port.perturb_bn_stats(net, NET_SEED + 1)
    return net


def batch(classes):
    return port.synthetic_batch(BATCH, H, W, seed=1, classes=classes)


def masks(net):
    return cases.dropout_masks(net, BATCH, seed=2)


def strided(n, k=16):
    """cases.grad_digest's k strided positions of an n-element tensor, spaced in float64: the PSP bottleneck's 18.9 M weights are
    beyond the integers float32 holds exactly."""
    return torch.linspace(0, n - 1, min(k, n), dtype=torch.float64).long()


def grad_digest(named_params):
    """cases.grad_digest (l2 norm, sum, strided samples of each gradient) with positions from `strided`."""
    out = {}
    for name, p in named_params:
        if p.grad is None:
            continue
        g = p.grad.detach().flatten().double()
        idx = strided(g.numel())
        out[name] = dict(norm=float(g.norm()), sum=float(g.sum()), samples=g[idx].float().clone(), idx=idx)
    return out


def param_samples(named_params):
    """The parameters at the gradient samples' positions."""
    return {name: p.detach().flatten()[strided(p.numel())].clone() for name, p in named_params}


def run_steps(net, criterion, images, labels):
    """STEPS training steps of `net` (train mode) -> list of per-step records."""
    opt = torch.optim.SGD([{'params': filter(lambda p: p.requires_grad, net.parameters()), 'initial_lr': LR}], LR,
                          momentum=MOMENTUM, weight_decay=WEIGHT_DECAY)                  # networks/kd_model.py:74
    net.train()
    recs = []
    for _ in range(STEPS):
        opt.zero_grad()
        preds = net(images)
        loss = criterion(preds, labels)
        loss.backward()
        rec = dict(loss=float(loss.detach()), logits=cases.sample_large(preds[0].detach().clone()), grads=grad_digest(net.named_parameters()))
        opt.step()
        rec["params"] = param_samples(net.named_parameters())
        recs.append(rec)
    return recs


def _ref_criterion(ref, ohem):
    if ohem:
        return ref.criterion.CriterionOhemDSN(255, OHEM_THRES, OHEM_KEEP)
    return ref.criterion.CriterionDSN()


def _port_criterion(ohem):
    if ohem:
        from tools import ohem_oracle
        return lambda preds, labels: ohem_oracle.ohem_dsn_loss(preds, labels, 255, OHEM_THRES, OHEM_KEEP)[0]
    return port.dsn_ce_loss


def ref_case(ref, name):
    arch, classes, ohem = CASES[name]
    src = build_net(arch, classes)
    P = ref.pspnet
    net = P.Res_pspnet(P.Bottleneck, [3, 4, 23, 3], classes) if arch == "resnet101" else P.Res_pspnet(P.BasicBlock, [2, 2, 2, 2], classes)
    net.load_state_dict(src.state_dict(), strict=True)
    for (holder, idx), m in zip(((net.pspmodule.bottleneck, 2), (net.dsn, 2)), masks(src)):
        cd = port.ChannelDropout(0.1); cd.injected = m
        holder[idx] = cd
    images, labels = batch(classes)
    out = io.StringIO()
    with _cpu_cuda_patch(), contextlib.redirect_stdout(out):
        recs = run_steps(net, _ref_criterion(ref, ohem), images, labels)
    res = dict(steps=recs, valid=int((labels != 255).sum()))
    if ohem:
        res["kept"] = [int(k) for k, _ in re.findall(r"Labels: (\d+) (\S+)", out.getvalue())]
        assert len(res["kept"]) == STEPS and all(0 < k < res["valid"] for k in res["kept"]), res["kept"]
    return res


def port_case(name):
    arch, classes, ohem = CASES[name]
    net = build_net(arch, classes)
    for d, m in zip(net.dropouts(), masks(net)):
        d.injected = m
    images, labels = batch(classes)
    return run_steps(net, _port_criterion(ohem), images, labels)


def compare(mine, gold):
    """-> (worst relative loss error, worst relative gradient-norm error) over the steps of a case."""
    loss = max(_rel(a["loss"], b["loss"]) for a, b in zip(mine, gold))
    grad = max(_rel(a["grads"][k]["norm"], v["norm"]) for a, b in zip(mine, gold) for k, v in b["grads"].items() if v["norm"] > 1e-6)
    return loss, grad


def main():
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count())
    gold = {}
    for name in CASES:
        t0 = time.time()
        gold[name] = ref_case(ref, name)
        loss, grad = compare(port_case(name), gold[name]["steps"])
        assert loss < 2e-4 and grad < 5e-3, (name, loss, grad)
        print(name, "loss", [round(s["loss"], 6) for s in gold[name]["steps"]], "kept", gold[name].get("kept"),
              "port: loss rel %.1e grad-norm rel %.1e" % (loss, grad), "%.1fs" % (time.time() - t0), flush=True)
    buf = io.BytesIO()
    torch.save(gold, buf)
    with gzip.open(GOLDEN, "wb") as f:
        f.write(buf.getvalue())
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")


def load():
    with gzip.open(GOLDEN, "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


if __name__ == "__main__":
    main()
