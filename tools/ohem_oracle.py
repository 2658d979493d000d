"""OHEM cross entropy (OhemCrossEntropy2d / CriterionOhemDSN, utils/criterion.py:11-90, 190-209): a torch CPU restatement
that uses scipy the way the reference does, the seeded cases, and the generator of tests/golden/ohem.pt.

The generator runs the UNMODIFIED reference classes on CPU (their `.cuda()` calls made the identity), pins the restatement
against them on the spot, and stores loss, threshold, kept count and sampled logit gradients per case, plus one golden
distillation step driven with CriterionOhemDSN:

    SKD_REFERENCE_ROOT=<reference checkout> python -m tools.ohem_oracle

TEST INFRASTRUCTURE ONLY.
"""
import contextlib
import io
import os
import re
import sys
import types

import numpy as np
import scipy.ndimage as nd
import torch
import torch.nn.functional as F

from oracle import cases, port

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ohem.pt")


# ----------------------------------------------------------------------------------------------------------- restatement
def grid_shape(H, W, factor):
    """scipy.ndimage.zoom's output size: round(in * (1 / factor)), Python rounding (half to even)."""
    return int(round(H * (1.0 / factor))), int(round(W * (1.0 / factor)))


def ohem_grid(prob, target, factor, ignore_label=255):
    """find_threshold's zoomed points (criterion.py:20-40): -> (pred (N, gh, gw) float32 with +inf where the zoomed label is
    ignored, zoomed labels (N, gh, gw) int64).  prob (N, C, H, W) and target (N, H, W) are numpy arrays."""
    zp = nd.zoom(prob, (1.0, 1.0, 1.0 / factor, 1.0 / factor), order=1)
    zt = nd.zoom(target, (1.0, 1.0 / factor, 1.0 / factor), order=0)
    valid = zt != ignore_label
    lab = np.where(valid, zt, 0)
    pred = np.take_along_axis(zp, lab[:, None], 1)[:, 0]
    return np.where(valid, pred, np.float32(np.inf)).astype(np.float32), zt.astype(np.int64)


def zoom_axis64(n_in, n_out, device=None):
    """scipy.ndimage.zoom's source coordinates along one axis (csrc/common.cuh zoom_ratio / zoom_axis), float64 torch ->
    (i0, i1, t, w0, nearest, outside): i0 / i1 the order-1 neighbours with weights w0 = 1 - t / t, `nearest` the order-0 source
    (floor(c + 0.5)), `outside` the points past n_in - 1 that mode 'constant' reads as 0."""
    r = (n_in - 1) / (n_out - 1) if n_out > 1 else 1.0
    c = torch.arange(n_out, dtype=torch.float64, device=device) * r
    outside = c > n_in - 1
    f = torch.floor(c)
    t = c - f
    i0 = f.long().clamp_max(n_in - 1)                          # (an outside point reads nothing: the clamp only keeps it indexable)
    i1 = (i0 + 1).clamp_max(n_in - 1)
    nearest = torch.floor(c + 0.5).long().clamp_max(n_in - 1)
    return i0, i1, t, 1.0 - t, nearest, outside


def ohem_grid64(prob, target, gh, gw, ignore_label=255):
    """ohem_grid in float64 torch on any device: prob (N, C, H, W) float64, target (N, H, W) int64 -> (pred (N, gh, gw) float64 with
    +inf where the zoomed label is ignored, zoomed labels (N, gh, gw) int64).  The four neighbours are weighted value * w_y * w_x
    and summed in scipy's order (common.cuh zoom_lerp); for float32 `prob` upcast to float64, pred.float() is scipy's output."""
    H, W = target.shape[1:]
    y0, y1, ty, wy, ny, oy = (a[:, None] for a in zoom_axis64(H, gh, prob.device))
    x0, x1, tx, wx, nx, ox = zoom_axis64(W, gw, prob.device)
    outside = oy | ox
    lab = torch.where(outside, 0, target[:, ny, nx])
    valid = lab != ignore_label
    idx = torch.where(valid, lab, 0).clamp(0, prob.shape[1] - 1)[:, None]
    p = [prob[:, :, a, b].gather(1, idx)[:, 0] for a, b in ((y0, x0), (y0, x1), (y1, x0), (y1, x1))]
    v = p[0] * wy * wx
    v = v + p[1] * wy * tx
    v = v + p[2] * ty * wx
    v = v + p[3] * ty * tx
    v = torch.where(outside, 0.0, v)
    return torch.where(valid, v, float("inf")), lab


def ohem_threshold(pred, min_kept, thresh):
    """criterion.py:27-48 on the grid values: 1.0 when min_kept >= valid, else thresh raised to the (min_kept-1)-th smallest."""
    valid = pred[np.isfinite(pred)]
    if min_kept >= valid.size:
        return 1.0
    threshold = thresh
    if min_kept > 0:
        k = min(valid.size, min_kept) - 1
        v = np.partition(valid, k)[k]
        if v > thresh:
            threshold = v
    return threshold


def ohem_ce_loss(predict, target, ignore_label=255, thresh=0.7, min_kept=100000, factor=8):
    """OhemCrossEntropy2d.forward at label resolution -> (loss, threshold (float32), kept pixel count)."""
    prob = torch.softmax(predict, 1)
    np_prob, np_target = prob.detach().numpy(), target.numpy()
    pred, _ = ohem_grid(np_prob, np_target, factor, ignore_label)
    thr = np.float32(ohem_threshold(pred, min_kept // (factor * factor), float(thresh)))
    valid = np_target != ignore_label
    p_lab = np.take_along_axis(np_prob, np.where(valid, np_target, 0)[:, None], 1)[:, 0]
    kept = valid & (p_lab <= thr)
    new_target = torch.from_numpy(np.where(kept, np_target, ignore_label)).long()
    return F.cross_entropy(predict, new_target, ignore_index=ignore_label), float(thr), int(kept.sum())


def ohem_dsn_loss(preds, target, ignore_index=255, thresh=0.7, min_kept=100000):
    """CriterionOhemDSN.forward: OHEM-CE(up(preds[0])) + 0.4 * CE(up(preds[1])) -> (loss, threshold, kept count)."""
    h, w = target.shape[1:]
    up0 = F.interpolate(preds[0], size=(h, w), mode="bilinear", align_corners=True)
    up1 = F.interpolate(preds[1], size=(h, w), mode="bilinear", align_corners=True)
    l1, thr, kept = ohem_ce_loss(up0, target, ignore_index, thresh, min_kept, 8)
    return l1 + 0.4 * F.cross_entropy(up1, target, ignore_index=ignore_index), thr, kept


# ----------------------------------------------------------------------------------------------------------- cases
# name: n, logits (h, w), labels (H, W), logits kind, thresh, min_kept, factor, standalone (OhemCrossEntropy2d at label size)
OHEM_CASES = {
    "dsn_65x129_512x1024": dict(n=2, hw=(65, 129), HW=(512, 1024), kind="random", thresh=0.7, min_kept=100000, factor=8),
    "dsn_confident_65x129": dict(n=2, hw=(65, 129), HW=(512, 1024), kind="confident", thresh=0.7, min_kept=100000, factor=8),
    "dsn_all_kept_64x64": dict(n=1, hw=(9, 9), HW=(64, 64), kind="random", thresh=0.7, min_kept=100000, factor=8),
    "dsn_zero_column_360x480": dict(n=2, hw=(46, 61), HW=(360, 480), kind="confident", thresh=0.7, min_kept=100000, factor=8),
    "dsn_half_way_36x44": dict(n=2, hw=(5, 6), HW=(36, 44), kind="random", thresh=0.7, min_kept=640, factor=8),
    "standalone_97x131_f4": dict(n=2, hw=(97, 131), HW=(97, 131), kind="random", thresh=0.7, min_kept=4000, factor=4,
                                 standalone=True),
}

# NetModel(ohem=True) against the reference modules driven with CriterionOhemDSN (batch 2 at 96 x 128, Pi + Pa).  A random-init
# student gives p[label] ~ 1/19 everywhere, so thresh 0.7 would keep every pixel: thresh 0 and min_kept = 192 * 64 put the
# threshold at the median of the 2 x 12 x 16 grid points, and about half of the valid pixels are dropped
OHEM_STEP = dict(name="ohem_pi_pa_96x128", batch=2, h=96, w=128, thresh=0.0, min_kept=192 * 64,
                 cfg=dict(pi=True, pa=True, ho=False, pool_scale=0.5))


def ohem_inputs(name):
    """-> (logits list [l0, l1] (l1 None for the standalone class), labels) of a case, seeded by its name."""
    c = OHEM_CASES[name]
    g = cases.seeded(sum(map(ord, name)))
    n, (h, w), (H, W) = c["n"], c["hw"], c["HW"]
    if c["kind"] == "confident":
        # smooth class regions: coarse logits upsampled to (h, w), scaled so that most pixels are sure of their label; the labels
        # are the argmax at label resolution, so p[label] is high away from region borders and the order statistic lies above 0.7
        coarse = torch.randn(n, 19, max(2, h // 16), max(2, w // 16), generator=g)
        l0 = F.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True) * 40 + 0.3 * torch.randn(n, 19, h, w, generator=g)
        labels = F.interpolate(l0, size=(H, W), mode="bilinear", align_corners=True).argmax(1)
    else:
        l0 = torch.randn(n, 19, h, w, generator=g) * (3.0 if c.get("standalone") else 2.0)
        labels = torch.randint(0, 19, (n, H, W), generator=g)
    labels[torch.rand(n, H, W, generator=g) < 0.05] = 255
    l1 = None if c.get("standalone") else torch.randn(n, 19, h, w, generator=g) * 2
    return [l0, l1], labels.contiguous()


def port_loss(name, preds, labels):
    c = OHEM_CASES[name]
    if c.get("standalone"):
        return ohem_ce_loss(preds[0], labels, 255, c["thresh"], c["min_kept"], c["factor"])
    return ohem_dsn_loss(preds, labels, 255, c["thresh"], c["min_kept"])


# ----------------------------------------------------------------------------------------------------------- generator
def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def _ref_criterion(ref, name):
    c = OHEM_CASES[name]
    if c.get("standalone"):
        return ref.criterion.OhemCrossEntropy2d(255, c["thresh"], c["min_kept"], c["factor"])
    return ref.criterion.CriterionOhemDSN(255, c["thresh"], c["min_kept"])


def criterion_golden(ref, name):
    from oracle.make_golden import _cpu_cuda_patch
    c = OHEM_CASES[name]
    preds, labels = ohem_inputs(name)
    for t in preds:
        if t is not None:
            t.requires_grad_(True)
    crit = _ref_criterion(ref, name)
    out = io.StringIO()
    with _cpu_cuda_patch(), contextlib.redirect_stdout(out):
        loss = crit(preds[0], labels) if c.get("standalone") else crit(preds, labels)
    printed = re.findall(r"Labels: (\d+) (\S+)", out.getvalue())
    grads = torch.autograd.grad(loss, [t for t in preds if t is not None])
    # the threshold as the reference object computes it, on the probabilities its forward thresholds
    ohem = crit if c.get("standalone") else crit.criterion1
    up0 = preds[0] if c.get("standalone") else F.interpolate(preds[0], size=labels.shape[1:], mode="bilinear", align_corners=True)
    thr = float(np.float32(ohem.find_threshold(torch.softmax(up0, 1).detach().numpy(), labels.numpy())))
    kept = int(printed[0][0]) if printed else 0
    if printed:
        assert float(np.float32(float(printed[0][1]))) == thr, (printed, thr)
    # the restatement, pinned now
    p_loss, p_thr, p_kept = port_loss(name, [None if t is None else t.detach() for t in preds], labels)
    loss = loss.detach()
    assert _rel(p_loss, loss) < 1e-6 and p_thr == thr and p_kept == kept, (name, float(p_loss), float(loss), p_thr, thr, p_kept, kept)
    rec = dict(loss=float(loss), threshold=thr, kept=kept, d_l0=cases.sample_large(grads[0].detach()))
    if len(grads) > 1:
        rec["d_l1"] = cases.sample_large(grads[1].detach())
    print("ohem", name, "loss %.6f threshold %.6f kept %d" % (rec["loss"], thr, kept))
    return rec


def step_golden(ref):
    """networks/kd_model.py:119-151 with the reference's modules and CriterionOhemDSN as the CE term."""
    from oracle import make_golden
    s = OHEM_STEP
    rc = types.SimpleNamespace(**vars(ref.criterion))
    rc.CriterionDSN = lambda: ref.criterion.CriterionOhemDSN(255, s["thresh"], s["min_kept"])
    r = types.SimpleNamespace(**vars(ref))
    r.criterion = rc
    out = io.StringIO()
    with make_golden._cpu_cuda_patch(), contextlib.redirect_stdout(out):
        gold = make_golden.step_goldens(r, {s["name"]: dict(batch=s["batch"], h=s["h"], w=s["w"], cfg=s["cfg"])}, check_port=False)
    gold = gold[s["name"]]
    (kept, thr), = re.findall(r"Labels: (\d+) (\S+)", out.getvalue())      # the reference's own print, once per call
    _, labels = port.synthetic_batch(s["batch"], s["h"], s["w"], seed=1)
    gold.update(kept=int(kept), threshold=float(np.float32(float(thr))), valid=int((labels != 255).sum()))
    assert 0 < gold["kept"] < gold["valid"], gold
    print("step", s["name"], {k: round(v, 6) for k, v in gold.items() if isinstance(v, (int, float))})
    return gold


def main():
    from oracle import refshim
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count())
    out = dict(criterion={name: criterion_golden(ref, name) for name in OHEM_CASES}, step=step_golden(ref))
    torch.save(out, GOLDEN)
    print("written", GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    sys.exit(main())
