"""Loss API of the reference (utils/criterion.py), same class names, constructor arguments, list-indexed inputs,
0-dim fp32 outputs with autograd history and error behaviour -- computed by hand-written sm_90a kernels.

  CriterionPixelWise                          utils/criterion.py:211-226
  CriterionPairWiseforWholeFeatAfterPool      utils/criterion.py:228-245   (alias: CriterionPairWise, the name the
                                              north star uses; it does not exist in the reference tree)
  CriterionDSN                                utils/criterion.py:168-188
  CriterionAdv / CriterionAdvForG             utils/criterion.py:122-166
  CriterionAdditionalGP                       utils/criterion.py:92-120
"""
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


class CriterionDSN(nn.Module):
    """DSN : two supervisions, loss1 + 0.4 * loss2."""

    def __init__(self, ignore_index=255, use_weight=True, reduce=True):
        super().__init__()
        self.ignore_index = ignore_index
        if not reduce:
            print("disabled the reduce.")

    def forward(self, preds, target):
        return Fn.DsnCrossEntropy.apply(preds[0], preds[1], target, self.ignore_index, 1.0, 0.4)


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
