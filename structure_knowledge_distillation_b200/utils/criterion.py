"""Loss API of the reference (utils/criterion.py), same class names, constructor arguments, list-indexed inputs,
0-dim fp32 outputs with autograd history and error behaviour -- computed by hand-written sm_90a kernels.

  CriterionPixelWise                          utils/criterion.py:211-226
  CriterionPairWiseforWholeFeatAfterPool      utils/criterion.py:228-245   (alias: CriterionPairWise, the name the
                                              north star uses; it does not exist in the reference tree)
  CriterionPairWiseLocal                      the pair-wise term over k x k node neighbourhoods (no reference source; it equals
                                              the class above when the window covers the grid at dilation 1)
  CriterionDSN                                utils/criterion.py:168-188
  CriterionCrossEntropy                       named at kd_model.py:79 (single head: the ESPNet-C student's task loss)
  OhemCrossEntropy2d                          utils/criterion.py:11-90
  CriterionOhemDSN                            utils/criterion.py:190-209
  CriterionAdv / CriterionAdvForG             utils/criterion.py:122-166
  CriterionAdditionalGP                       utils/criterion.py:92-120
  CriterionAT / CriterionMimic                the feature-level baselines the paper compares with (no reference source: attention
                                              transfer after Zagoruyko & Komodakis, MIMIC after Li et al.)
  CriterionCWD                                channel-wise distillation (Shu et al., ICCV 2021), the structured term's usual
                                              competitor (no reference source)
  CriterionIFV                                intra-class feature variation distillation (Wang et al., ECCV 2020), structured KD's
                                              successor on the same setting (no reference source)

The OHEM criteria follow the reference's threshold rule (scipy's zoom to a 1/factor grid with its exact arithmetic, the order
statistic, pixels with p[label] <= threshold kept) but compute it on the device, without the reference's host round trip.
Differences, on purpose:
  * no `Labels: <kept> <threshold>` print per call; the criterion keeps `last_threshold` and `last_kept` as device tensors;
  * `weight` is ignored (so is it in the reference);
  * with several ranks each rank thresholds its own shard (the reference's per-replica criterion semantics);
  * when no pixel is kept the loss is NaN, as torch's cross entropy returns, and the gradient is zero.
"""
import math
import numbers

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


class CriterionPairWiseLocal(nn.Module):
    """Local pair-wise loss: pooling and normalisation as CriterionPairWiseforWholeFeatAfterPool's, but node i = (y, x) of the pooled
    h x w grid is compared only with the nodes j = (y + t * dilation, x + u * dilation), t, u in -r..r (r = (window - 1) / 2), that lie
    inside the grid, j = i included: L = sum_n sum_i sum_{j in W(i)} (a^T_ij - a^S_ij)^2 / (N * P), P the connected ordered pairs per
    image.  With dilation 1 and a window covering the grid it is the fully connected term.  pool_scale = 1 / h gives one node per pixel
    (when w < 2h)."""

    def __init__(self, scale, feat_ind, window, dilation=1):
        super().__init__()
        self.feat_ind = feat_ind
        self.scale = scale
        self.window = _check_pa_window("pa_window", window)
        self.dilation = _check_pa_dilation("pa_dilation", dilation)

    def forward(self, preds_S, preds_T):
        feat_S = preds_S[self.feat_ind]
        feat_T = preds_T[self.feat_ind].detach()
        total_w, total_h = feat_T.shape[2], feat_T.shape[3]
        patch_w, patch_h = int(total_w * self.scale), int(total_h * self.scale)
        return Fn.PairWiseLocalLoss.apply(feat_S, feat_T, patch_w, patch_h, self.window, self.dilation)


PA_WINDOW_MAX, PA_DILATION_MAX = 15, 8

PA_LEVELS_MAX = 5         # preds[-1] .. preds[-5]: x1, x2, x3, x4 and the PSP features of every student


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
    _check_level_count("lambda_pa / pool_scale lists", len(lam))
    levels = []
    for ind, (l, s) in enumerate(zip(lam, scale)):
        try:
            l, s = float(l), float(s)
        except (TypeError, ValueError):
            raise ValueError("pair-wise level %d: lambda_pa and pool_scale must be numbers (got %r, %r)" % (ind, l, s)) from None
        _check_level_weight("pair-wise level %d: lambda_pa" % ind, l)
        if not (math.isfinite(s) and 0 < s <= 1):
            raise ValueError("pair-wise level %d: pool_scale must be in (0, 1] (got %r)" % (ind, s))
        levels.append((l, s))
    return levels


def _is_int(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def _check_pa_window(what, k):
    if not _is_int(k) or k % 2 == 0 or not 3 <= k <= PA_WINDOW_MAX:
        raise ValueError("%s must be None or an odd int in 3..%d (got %r)" % (what, PA_WINDOW_MAX, k))
    return int(k)


def _check_pa_dilation(what, d):
    if not _is_int(d) or not 1 <= d <= PA_DILATION_MAX:
        raise ValueError("%s must be an int in 1..%d (got %r)" % (what, PA_DILATION_MAX, d))
    return int(d)


def check_pa_windows(args):
    """`args.pa_window` / `args.pa_dilation` of NetModel, validated before any device work against the form of `lambda_pa`.  The
    defaults (None and 1) keep every pair-wise level fully connected -> None.  Otherwise they follow lambda_pa: two scalars when it is
    a scalar -> (window, dilation) of the single term on preds[-5], or None when the window is None; two lists of its length when it is a
    list -> [(window or None, dilation)] per level, None keeping that level fully connected.  In the list form a default left as the
    scalar (pa_window=None or pa_dilation=1) stands for every level.  A window is an odd int in 3..15, a dilation an int in 1..8, and a
    fully connected level takes dilation 1; anything else raises ValueError naming the field and the level."""
    win, dil = getattr(args, "pa_window", None), getattr(args, "pa_dilation", 1)
    win_list, dil_list = isinstance(win, (list, tuple)), isinstance(dil, (list, tuple))
    if not win_list and not dil_list and win is None and _is_int(dil) and dil == 1:
        return None
    lam = getattr(args, "lambda_pa", 0.5)
    if not isinstance(lam, (list, tuple)):
        if win_list or dil_list:
            raise ValueError("pa_window and pa_dilation must be scalars when lambda_pa is a scalar (got %r and %r)" % (win, dil))
        dil = _check_pa_dilation("pa_dilation", dil)
        if win is None:
            raise ValueError("pa_dilation %r needs a local window: pa_window is None (the fully connected term)" % (dil,))
        return _check_pa_window("pa_window", win), dil
    n = len(lam)
    if win is None and not win_list:
        win = [None] * n
    elif not win_list:
        raise ValueError("pa_window must be a list of %d entries when lambda_pa is a list (got %r)" % (n, win))
    if _is_int(dil) and dil == 1 and not dil_list:
        dil = [1] * n
    elif not dil_list:
        raise ValueError("pa_dilation must be a list of %d entries when lambda_pa is a list (got %r)" % (n, dil))
    if len(win) != n or len(dil) != n:
        raise ValueError("pa_window and pa_dilation lists must have %d entries like lambda_pa (got %d and %d)" % (n, len(win), len(dil)))
    levels = []
    for ind, (k, d) in enumerate(zip(win, dil)):
        d = _check_pa_dilation("pair-wise level %d: pa_dilation" % ind, d)
        if k is None:
            if d != 1:
                raise ValueError("pair-wise level %d: pa_dilation %d needs a local window (pa_window is None)" % (ind, d))
        else:
            k = _check_pa_window("pair-wise level %d: pa_window" % ind, k)
        levels.append((k, d))
    return levels


def _check_level_count(what, n):
    if not 1 <= n <= PA_LEVELS_MAX:
        raise ValueError("%s must have 1..%d entries (got %d)" % (what, PA_LEVELS_MAX, n))


def _check_level_weight(what, w):
    if not math.isfinite(w) or w < 0:
        raise ValueError("%s must be finite and >= 0 (got %r)" % (what, w))


def check_feature_levels(args, name, term, default):
    """`args.<name>` (lambda_at / lambda_mimic) of NetModel, validated before any device work -> [(feat_ind, weight)]: a scalar is
    one term on preds[-5] (the PSP features); a list (or tuple) of L weights, 1 <= L <= 5, puts level `ind` on preds[-(ind + 1)] as
    the pair-wise levels do (check_pa_levels).  Each weight finite and >= 0 (0 skips the level); anything else raises ValueError
    naming `term`."""
    lam = getattr(args, name, default)
    if not isinstance(lam, (list, tuple)):
        try:
            lam = float(lam)
        except (TypeError, ValueError):
            raise ValueError("%s must be a number or a list of numbers (got %r)" % (name, lam)) from None
        _check_level_weight(name, lam)
        return [(-5, lam)]
    _check_level_count(name + " list", len(lam))
    levels = []
    for ind, l in enumerate(lam):
        try:
            l = float(l)
        except (TypeError, ValueError):
            raise ValueError("%s level %d: %s must be a number (got %r)" % (term, ind, name, l)) from None
        _check_level_weight("%s level %d: %s" % (term, ind, name), l)
        levels.append((-(ind + 1), l))
    return levels


def pair_wise_level_criteria(levels, windows=None):
    """One CriterionPairWiseforWholeFeatAfterPool per level of check_pa_levels(), level `ind` on preds[-(ind + 1)]
    (kd_model.py:81); a CriterionPairWiseLocal instead where `windows` (check_pa_windows()'s list) gives the level a window."""
    windows = windows or [(None, 1)] * len(levels)
    return [CriterionPairWiseforWholeFeatAfterPool(scale=s, feat_ind=-(ind + 1)) if k is None else
            CriterionPairWiseLocal(scale=s, feat_ind=-(ind + 1), window=k, dilation=d)
            for ind, ((_, s), (k, d)) in enumerate(zip(levels, windows))]


class CriterionAT(nn.Module):
    """Attention transfer (Zagoruyko & Komodakis) between preds_S[feat_ind] and preds_T[feat_ind]: mean over N*H*W of
    (at(S) - at(T))^2 with at(x) = F.normalize(x.pow(2).mean(1).view(N, -1)) (p = 2).  Channel-agnostic: the two widths may differ."""

    def __init__(self, feat_ind):
        super().__init__()
        self.feat_ind = feat_ind

    def forward(self, preds_S, preds_T):
        return Fn.AttentionTransferLoss.apply(preds_S[self.feat_ind], preds_T[self.feat_ind].detach())


class CriterionMimic(nn.Module):
    """MIMIC (Li et al.): F.mse_loss(adapter(preds_S[feat_ind]), preds_T[feat_ind]), `adapter` a 1x1 convolution with bias from the
    student's to the teacher's width (networks/pspnet_combine.Conv2d, on the wgmma kernels)."""

    def __init__(self, feat_ind, adapter):
        super().__init__()
        self.feat_ind = feat_ind
        self.adapter = adapter

    def forward(self, preds_S, preds_T):
        return Fn.MseLoss.apply(self.adapter(preds_S[self.feat_ind]), preds_T[self.feat_ind].detach())


class CriterionCWD(nn.Module):
    """Channel-wise distillation (Shu et al.): tau^2 / (N*C) * sum over (n, c) of KL(softmax_HW(T / tau) || softmax_HW(S / tau)), S =
    preds_S[feat_ind] (through `adapter`, a 1x1 convolution from the student's to the teacher's width, when given) and T =
    preds_T[feat_ind] detached, on one grid (Fn.ChannelWiseLoss)."""

    def __init__(self, feat_ind, tau, adapter=None):
        super().__init__()
        self.feat_ind = feat_ind
        self.tau = float(tau)
        self.adapter = adapter

    def forward(self, preds_S, preds_T):
        s = preds_S[self.feat_ind]
        if self.adapter is not None:
            s = self.adapter(s)
        return Fn.ChannelWiseLoss.apply(s, preds_T[self.feat_ind].detach(), self.tau)


def check_cwd_args(args):
    """NetModel's channel-wise distillation options, validated before any device work -> (lambda_cwd, cwd_tau, feature levels):
    lambda_cwd a number, finite and >= 0 (the logit term's weight, 0 turns it off); cwd_tau a number, finite and > 0; lambda_cwd_feat
    None (no feature term, []) or check_feature_levels()' form.  Anything else raises ValueError naming the field."""
    lam = getattr(args, "lambda_cwd", 3.0)
    if isinstance(lam, (list, tuple)):
        raise ValueError("lambda_cwd must be a number, the weight of the logit term (got the list %r; feature levels go in "
                         "lambda_cwd_feat)" % (lam,))
    try:
        lam = float(lam)
    except (TypeError, ValueError):
        raise ValueError("lambda_cwd must be a number (got %r)" % (lam,)) from None
    _check_level_weight("lambda_cwd", lam)
    tau = getattr(args, "cwd_tau", 4.0)
    try:
        tau = float(tau)
    except (TypeError, ValueError):
        raise ValueError("cwd_tau must be a number (got %r)" % (tau,)) from None
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError("cwd_tau must be finite and > 0 (got %r)" % (tau,))
    if getattr(args, "lambda_cwd_feat", None) is None:
        return lam, tau, []
    return lam, tau, check_feature_levels(args, "lambda_cwd_feat", "CWD", None)


class CriterionIFV(nn.Module):
    """Intra-class feature variation distillation (Wang et al., IFVD) of preds_S[feat_ind] against preds_T[feat_ind] detached, on one
    grid, with the step's (N, H, W) int64 labels taken down to that grid by nearest (Fn.IntraClassVariationLoss): per image and class in
    [0, classes_num) the prototype of each map, then the mean over all pixels of (cos(f_S, P_S) - cos(f_T, P_T))^2.  `ignore_index`
    names the unlabelled pixels' label; like every label outside [0, classes_num) they add nothing, so it must lie outside that range."""

    def __init__(self, feat_ind, classes_num, ignore_index=255):
        super().__init__()
        if not 1 <= int(classes_num) <= 255:
            raise ValueError("IFV needs 1 <= classes_num <= 255 (got %r)" % (classes_num,))
        if 0 <= ignore_index < classes_num:
            raise ValueError("IFV: ignore_index %r is one of the %d classes" % (ignore_index, classes_num))
        self.feat_ind = feat_ind
        self.classes_num = int(classes_num)
        self.ignore_index = ignore_index

    def forward(self, preds_S, preds_T, labels):
        return Fn.IntraClassVariationLoss.apply(preds_S[self.feat_ind], preds_T[self.feat_ind].detach(), labels, self.classes_num)


def check_ifv_args(args):
    """NetModel's IFV options, validated before any device work -> [(feat_ind, weight)] of lambda_ifv (check_feature_levels()' form),
    or [] while the term is off.  `ifv` must be True or False (a string such as "False" would otherwise read as on)."""
    on = getattr(args, "ifv", False)
    if not (isinstance(on, (bool, int)) and on in (0, 1)):
        raise ValueError("ifv must be True or False (got %r)" % (on,))
    levels = check_feature_levels(args, "lambda_ifv", "IFV", 200.0)
    return levels if on else []


def feature_level_criteria(levels, make):
    """One criterion `make(feat_ind)` per level of check_feature_levels() with a non-zero weight, None for the others."""
    return [make(i) if w != 0.0 else None for i, w in levels]


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
