"""SAGAN discriminator of the holistic (Ho) loss -- same classes, constructor arguments, state-dict names and [out, p1, p2]
output as networks/sagan_models.py:9-41,105-168, executed by hand-written sm_90a kernels (networks/sagan_engine.py,
csrc/disc.cu, wgmma convolutions): no torch operator, cuDNN or cuBLAS call on the forward, backward or WGAN-GP path.

The modules below are parameter containers with the reference's names; `Discriminator.forward` is one autograd node
(`DiscriminatorFn`).  Differences that are visible to a caller:
  * the attention maps p1 / p2 are returned non-differentiable;
  * `imsize` no longer gates the fourth block (sagan_models.py:131-136 leaves `self.l4` undefined unless imsize == 65 and
    forward() then fails): l4 is always built, and the 4x4 "last" conv uses the top-left window of its kernel when the map it
    sees is smaller than 4x4 (360x480 crops -> 46x61 logits -> 2x3 map; SURVEY.md §8-f2).  With 65-pixel logits the
    behaviour is the reference's.
"""
import torch
import torch.nn as nn

from .pspnet_combine import Conv2d
from .sagan_engine import DiscEngine, DiscriminatorFn
from .spectral import SpectralNorm


class Self_Attn(nn.Module):
    """Self attention layer: softmax(Q^T K) without 1/sqrt(d), out = gamma * (V A^T) + x, gamma initialised to 0
    (sagan_models.py:9-41).  query/key/value 1x1 convolutions are one (2d+C) x C GEMM on wgmma; the core is csrc/disc.cu."""

    def __init__(self, in_dim, activation=None):
        super().__init__()
        self.chanel_in, self.activation = in_dim, activation
        self.query_conv = Conv2d(in_dim, in_dim // 8, 1)
        self.key_conv = Conv2d(in_dim, in_dim // 8, 1)
        self.value_conv = Conv2d(in_dim, in_dim, 1)
        self.gamma = nn.Parameter(torch.zeros(1))

    def forward(self, x):
        from .sagan_engine import SelfAttnFn
        return SelfAttnFn.apply(self, x, *[p for p in self.parameters()])


class Discriminator(nn.Module):
    """Discriminator, Auxiliary Classifier."""

    def __init__(self, preprocess_GAN_mode, input_channel, batch_size=64, image_size=64, conv_dim=64):
        super().__init__()
        self.imsize = image_size
        d = conv_dim
        self.l1 = nn.Sequential(SpectralNorm(Conv2d(input_channel, d, 4, 2, 1)), nn.LeakyReLU(0.1))
        self.l2 = nn.Sequential(SpectralNorm(Conv2d(d, d * 2, 4, 2, 1)), nn.LeakyReLU(0.1))
        self.l3 = nn.Sequential(SpectralNorm(Conv2d(d * 2, d * 4, 4, 2, 1)), nn.LeakyReLU(0.1))
        self.l4 = nn.Sequential(SpectralNorm(Conv2d(d * 4, d * 8, 4, 2, 1)), nn.LeakyReLU(0.1))
        self.n_sn_layers = 4
        self.last = nn.Sequential(Conv2d(d * 8, 1, 4))
        self.attn1 = Self_Attn(d * 4, 'relu')
        self.attn2 = Self_Attn(d * 8, 'relu')
        self.preprocess_mode = preprocess_GAN_mode
        if preprocess_GAN_mode == 1:
            self.preprocess_additional = nn.BatchNorm2d(input_channel)       # parameter / buffer container; math in csrc/disc.cu
        elif preprocess_GAN_mode == 2:
            self.preprocess_additional = nn.Tanh()
        elif preprocess_GAN_mode == 3:
            self.preprocess_additional = lambda x: 2 * (x / 255 - 0.5)
        else:
            raise ValueError('preprocess_GAN_mode should be 1:bn or 2:tanh or 3:-1 - 1')
        self.sn_names = ["l1.0.module", "l2.0.module", "l3.0.module", "l4.0.module"]
        self.engine = DiscEngine(self)
        # NetModel switches these: the generator step needs only d out / d logits (kd_model.py:147-150 followed by
        # D_solver.zero_grad() at :154 discards D's gradients of that pass); the D step accumulates straight into the flat
        # gradient buffer of FlatSGD instead of returning ~25 tensors for autograd to add one by one
        self.skip_param_grads = False
        self.accumulate_into_grad = False

    @property
    def grad_names(self):
        return [n for n, p in self.named_parameters() if p.requires_grad]

    def forward(self, x):
        params = [p for p in self.parameters() if p.requires_grad]
        return list(DiscriminatorFn.apply(self, x, *params))
