"""Loss API of the reference (utils/criterion.py), same class names, constructor arguments, list-indexed inputs,
0-dim fp32 outputs with autograd history and error behaviour -- computed by hand-written sm_90a kernels.

  CriterionPixelWise                          utils/criterion.py:211-226
  CriterionPairWiseforWholeFeatAfterPool      utils/criterion.py:228-245   (alias: CriterionPairWise, the name the
                                              north star uses; it does not exist in the reference tree)
  CriterionDSN                                utils/criterion.py:168-188
  CriterionCrossEntropy                       named at kd_model.py:79 (single head: the ESPNet-C student's task loss)
  OhemCrossEntropy2d                          utils/criterion.py:11-90
  CriterionOhemDSN                            utils/criterion.py:190-209
  CriterionAdv / CriterionAdvForG             utils/criterion.py:122-166
  CriterionAdditionalGP                       utils/criterion.py:92-120

The OHEM criteria follow the reference's threshold rule (scipy's zoom to a 1/factor grid with its exact arithmetic, the order
statistic, pixels with p[label] <= threshold kept) but compute it on the device, without the reference's host round trip.
Differences, on purpose:
  * no `Labels: <kept> <threshold>` print per call; the criterion keeps `last_threshold` and `last_kept` as device tensors;
  * `weight` is ignored (so is it in the reference);
  * with several ranks each rank thresholds its own shard (the reference's per-replica criterion semantics);
  * when no pixel is kept the loss is NaN, as torch's cross entropy returns, and the gradient is zero.
"""
import math

import torch
import torch.nn as nn

from .. import functions as Fn
from ..networks.sagan_engine import AdvLossFn, GradientPenaltyFn


class CriterionPixelWise(nn.Module):
    def __init__(self, ignore_index=255, use_weight=True, reduce=True):
        super().__init__()
        self.ignore_index = ignore_index

    def forward(self, preds_S, preds_T):
        assert preds_S[0].shape == preds_T[0].shape, 'the output dim of teacher and student differ'
        return Fn.PixelWiseLoss.apply(preds_S[0], preds_T[0].detach())


class CriterionPairWiseforWholeFeatAfterPool(nn.Module):
    def __init__(self, scale, feat_ind):
        """inter pair-wise loss from inter feature maps"""
        super().__init__()
        self.feat_ind = feat_ind
        self.scale = scale

    def forward(self, preds_S, preds_T):
        feat_S = preds_S[self.feat_ind]
        feat_T = preds_T[self.feat_ind].detach()
        total_w, total_h = feat_T.shape[2], feat_T.shape[3]
        patch_w, patch_h = int(total_w * self.scale), int(total_h * self.scale)      # criterion.py:241-242
        return Fn.PairWiseLoss.apply(feat_S, feat_T, patch_w, patch_h)


CriterionPairWise = CriterionPairWiseforWholeFeatAfterPool

PA_LEVELS_MAX = 5          # preds[-1] .. preds[-5]: x1, x2, x3, x4 and the PSP features of every student


def check_pa_levels(args):
    """`args.lambda_pa` / `args.pool_scale` of NetModel, validated before any device work.  Two scalars (the defaults): None, the
    single pair-wise term on preds[-5].  Two lists (or tuples) of equal length L, 1 <= L <= 5: the multi-level form of the
    reference's kd_model.py:81,137-143, returned as [(lambda, scale), ...] where entry `ind` distils preds[-(ind + 1)] -- 0 is x1
    (layer1), 1 x2, 2 x3, 3 x4, 4 the PSP features; so a one-entry list distils x1, not preds[-5].  Each lambda finite and >= 0
    (0 skips the level), each scale in (0, 1]; anything else raises ValueError."""
    lam, scale = getattr(args, "lambda_pa", 0.5), getattr(args, "pool_scale", 0.5)
    lam_list, scale_list = isinstance(lam, (list, tuple)), isinstance(scale, (list, tuple))
    if not lam_list and not scale_list:
        return None
    if lam_list != scale_list:
        raise ValueError("lambda_pa and pool_scale must both be scalars or both be lists (got %r and %r)" % (lam, scale))
    if len(lam) != len(scale):
        raise ValueError("lambda_pa and pool_scale lists differ in length (%d and %d)" % (len(lam), len(scale)))
    if not 1 <= len(lam) <= PA_LEVELS_MAX:
        raise ValueError("lambda_pa / pool_scale lists must have 1..%d entries (got %d)" % (PA_LEVELS_MAX, len(lam)))
    levels = []
    for ind, (l, s) in enumerate(zip(lam, scale)):
        try:
            l, s = float(l), float(s)
        except (TypeError, ValueError):
            raise ValueError("pair-wise level %d: lambda_pa and pool_scale must be numbers (got %r, %r)" % (ind, l, s)) from None
        if not math.isfinite(l) or l < 0:
            raise ValueError("pair-wise level %d: lambda_pa must be finite and >= 0 (got %r)" % (ind, l))
        if not (math.isfinite(s) and 0 < s <= 1):
            raise ValueError("pair-wise level %d: pool_scale must be in (0, 1] (got %r)" % (ind, s))
        levels.append((l, s))
    return levels


def pair_wise_level_criteria(levels):
    """One CriterionPairWiseforWholeFeatAfterPool per level of check_pa_levels(), level `ind` on preds[-(ind + 1)]
    (kd_model.py:81)."""
    return [CriterionPairWiseforWholeFeatAfterPool(scale=s, feat_ind=-(ind + 1)) for ind, (_, s) in enumerate(levels)]


def check_class_weights(weight, classes_num=None):
    """-> the class weights as a float32 CPU tensor, or None.  `weight` is a 1-D sequence or tensor of non-negative finite floats,
    not all zero, with `classes_num` entries when that is given; anything else raises ValueError."""
    if weight is None:
        return None
    try:
        w = torch.as_tensor(weight.detach().cpu() if torch.is_tensor(weight) else weight, dtype=torch.float64)
    except (TypeError, ValueError, RuntimeError) as e:
        raise ValueError("class weights must be a 1-D sequence of floats (%s)" % e) from None
    if w.dim() != 1 or w.numel() == 0:
        raise ValueError("class weights must be a non-empty 1-D sequence (got shape %s)" % (tuple(w.shape),))
    if classes_num is not None and w.numel() != int(classes_num):
        raise ValueError("class weights have %d entries for %d classes" % (w.numel(), int(classes_num)))
    if not bool(torch.isfinite(w).all()) or bool((w < 0).any()):
        raise ValueError("class weights must be finite and non-negative (got %s)" % w.tolist())
    if not bool((w > 0).any()):
        raise ValueError("class weights are all zero")
    return w.float()


def check_task_loss_weights(args):
    """`args.class_weights` (default None) of NetModel / SegModel, validated against `args.classes_num` before any device work.
    OHEM ignores class weights (so does the reference's OhemCrossEntropy2d), so asking for both raises ValueError."""
    weight = getattr(args, "class_weights", None)
    if weight is not None and getattr(args, "ohem", False):
        raise ValueError("class_weights cannot be combined with ohem=True (the OHEM cross entropy is unweighted)")
    return check_class_weights(weight, args.classes_num)


class _WeightedCE(nn.Module):
    """Holds the optional class-weight table of the task losses: copied to the device once, at `.to(device)` or at the first call."""

    def __init__(self, weight):
        super().__init__()
        self.register_buffer("weight", check_class_weights(weight))

    def _weight(self, logits):
        w = self.weight
        if w is None:
            return None
        if w.numel() != logits.shape[1]:
            raise ValueError("class weights have %d entries for %d classes" % (w.numel(), logits.shape[1]))
        if w.device != logits.device:
            self.weight = w = w.to(logits.device)
        return w


class CriterionDSN(_WeightedCE):
    """DSN : two supervisions, loss1 + 0.4 * loss2.  `weight`: optional per-class weights of both cross entropies, as
    torch.nn.CrossEntropyLoss(weight=...) applies them (a weighted mean with the heads' common denominator sum_i weight[y_i])."""

    def __init__(self, ignore_index=255, use_weight=True, reduce=True, weight=None):
        super().__init__(weight)
        self.ignore_index = ignore_index
        if not reduce:
            print("disabled the reduce.")

    def forward(self, preds, target):
        return Fn.DsnCrossEntropy.apply(preds[0], preds[1], target, self.ignore_index, 1.0, 0.4, self._weight(preds[0]))


class CriterionCrossEntropy(_WeightedCE):
    """Single-head cross entropy, CE(up(preds[0])) with bilinear align_corners to the label size, mean over the valid pixels (the
    class the reference names for students without an auxiliary head, kd_model.py:79): the task loss of the ESPNet-C student.
    `weight`: optional per-class weights, as torch.nn.CrossEntropyLoss(weight=...) applies them."""

    def __init__(self, ignore_index=255, use_weight=True, reduce=True, weight=None):
        super().__init__(weight)
        self.ignore_index = ignore_index

    def forward(self, preds, target):
        return Fn.DsnCrossEntropy.apply(preds[0], None, target, self.ignore_index, 1.0, 0.0, self._weight(preds[0]))


class OhemCrossEntropy2d(nn.Module):
    """Cross entropy over the hard pixels only: those whose softmax probability of the label is <= a threshold found on a
    1/`factor` grid (at least ~`min_kept` pixels, never fewer than those under `thresh`).  `predict` is (n, c, H, W) at label
    resolution.  Limit: the fused loss kernel holds one row of `predict` in shared memory, so W may be at most 1 483 columns with
    19 classes (about 760 with 32); wider inputs (full-size 1024x2048 Cityscapes maps) raise RuntimeError ("source width too
    large").  CriterionOhemDSN has no such limit in practice: it reads the low-resolution logits (65x129 at 512x1024)."""

    def __init__(self, ignore_label=255, thresh=0.7, min_kept=100000, factor=8):
        super().__init__()
        self.ignore_label = ignore_label
        self.thresh = float(thresh)
        self.min_kept = int(min_kept)
        self.factor = factor
        self.last_threshold = None
        self.last_kept = None

    def forward(self, predict, target, weight=None):
        assert not target.requires_grad
        loss, self.last_threshold, self.last_kept = Fn.OhemDsnCrossEntropy.apply(
            predict, None, target, self.ignore_label, self.thresh, self.min_kept, self.factor, 1.0, 0.0)
        return loss


class CriterionOhemDSN(nn.Module):
    """DSN with OHEM on the main head: OhemCrossEntropy2d(up(preds[0])) + 0.4 * CE(up(preds[1])), bilinear align_corners to the
    label size, fused so that neither upsampled logit map is materialised."""

    def __init__(self, ignore_index=255, thresh=0.7, min_kept=100000, use_weight=True, reduce=True):
        super().__init__()
        self.ignore_index = ignore_index
        self.criterion1 = OhemCrossEntropy2d(ignore_index, thresh, min_kept)
        self.last_threshold = None
        self.last_kept = None

    def forward(self, preds, target):
        assert not target.requires_grad
        c = self.criterion1
        loss, self.last_threshold, self.last_kept = Fn.OhemDsnCrossEntropy.apply(
            preds[0], preds[1], target, self.ignore_index, c.thresh, c.min_kept, c.factor, 1.0, 0.4)
        c.last_threshold, c.last_kept = self.last_threshold, self.last_kept
        return loss


class CriterionAdvForG(nn.Module):
    def __init__(self, adv_type):
        super().__init__()
        if (adv_type != 'wgan-gp') and (adv_type != 'hinge'):
            raise ValueError('adv_type should be wgan-gp or hinge')
        self.adv_loss = adv_type

    def forward(self, d_out_S, d_out_S_no_use=None):
        """-mean(D(S)) for both adversarial types (criterion.py:129-137)."""
        return AdvLossFn.apply(None, d_out_S[0], 2)


class CriterionAdv(nn.Module):
    def __init__(self, adv_type):
        super().__init__()
        if (adv_type != 'wgan-gp') and (adv_type != 'hinge'):
            raise ValueError('adv_type should be wgan-gp or hinge')
        self.adv_loss = adv_type

    def forward(self, d_out_S, d_out_T):
        assert d_out_S[0].shape == d_out_T[0].shape, 'the output dim of D with teacher and student as input differ'
        return AdvLossFn.apply(d_out_T[0], d_out_S[0], 0 if self.adv_loss == 'wgan-gp' else 1)


class CriterionAdditionalGP(nn.Module):
    """WGAN-GP penalty lambda * mean((|d D(x)/dx|_2 - 1)^2) at x = alpha real + (1 - alpha) fake (criterion.py:98-120).
    The reference differentiates it by double backward through D; here the value and the parameter gradient come from the
    discriminator engine's first-order chain / tangent pass / joint reverse pass (networks/sagan_engine.py) -- `D_net` must be
    this package's Discriminator."""

    def __init__(self, D_net, lambda_gp):
        super().__init__()
        self.D = D_net
        self.lambda_gp = lambda_gp
        self.alpha = None            # optional injected (N,1,1,1) interpolation weights (parity tests)

    def forward(self, d_in_S, d_in_T):
        assert d_in_S[0].shape == d_in_T[0].shape, 'the output dim of D with teacher and student as input differ'
        D = self.D
        if not hasattr(D, "engine"):
            raise TypeError("CriterionAdditionalGP needs structure_knowledge_distillation_b200's Discriminator (no autograd double backward here)")
        real, fake = d_in_T[0].detach(), d_in_S[0].detach()
        alpha = self.alpha if self.alpha is not None else torch.rand(real.size(0), 1, 1, 1, device=real.device)
        x = torch.lerp(fake, real, alpha.to(real.dtype))               # alpha * real + (1 - alpha) * fake
        return GradientPenaltyFn.apply(D, x, float(self.lambda_gp), *[p for p in D.parameters() if p.requires_grad])
