"""`SegModel` -- a segmentation training step with no teacher and no discriminator, on the same sm_90a kernels as NetModel's student.

It trains what NetModel distills from: the PSPNet-ResNet101 teacher (`seg_model='resnet101'`, the default), for a class count or a crop
size nobody publishes a checkpoint for, and every student kind without distillation (the reference's "baseline" row: ResNet18-PSP
trained on the task loss alone).  The step API and its machinery are NetModel's, from StepModel (networks/step_model.py): set_input,
forward, backward, optimize_parameters, adjust_learning_rate, lr_poly, print_info, save_ckpt, evalute_model; .model .G_solver .preds
.G_loss .mc_G_loss.  So a train_and_eval.py-style loop drives it unchanged, and what save_ckpt writes loads through load_T_model as
NetModel's teacher (`T_ckpt_path`).  SegModel adds the split-precision policy of the ResNets.
"""
import logging

from .. import ops
from ..utils.utils import load_seg_model
from .pspnet_combine import Conv2d
from .step_model import SEG_MODELS, StepModel, _LazyScalar, _arg, build_seg_network

# Which convolutions of a PSP ResNet run their training forward in split-precision 3xTF32 (DESIGN.md §4, "The teacher in training"):
#   'early':  the stem, layer1 and layer2 -- the ResNet18 student's flags (ResNet.set_precise_early_layers);
#   'layer3': those plus layer3;
#   'all':    every convolution.
PRECISION_POLICIES = ("early", "layer3", "all")
DEFAULT_PRECISION = {"resnet101": "all", "resnet18": "early"}


def set_precision_policy(net, policy):
    """Sets `Conv2d.precise` on every convolution of a Res_pspnet network according to `policy` (PRECISION_POLICIES)."""
    if policy not in PRECISION_POLICIES:
        raise ValueError("precision policy must be one of %s (got %r)" % (PRECISION_POLICIES, policy))
    convs = [m for m in net.modules() if isinstance(m, Conv2d)]
    for m in convs:
        m.precise = False
    if policy == "all":
        for m in convs:
            m.precise = True
        return
    net.set_precise_early_layers(True)
    if policy == "layer3":
        for m in net.layer3.modules():
            if isinstance(m, Conv2d):
                m.precise = True


class SegModel(StepModel):
    def name(self):
        return 'seg'

    def __init__(self, args):
        super().__init__(args)
        self._check_kind("seg_model", "resnet101", SEG_MODELS)
        self._check_device()
        model = build_seg_network(self.kind, args.classes_num, args)
        if self.kind in DEFAULT_PRECISION:
            set_precision_policy(model, str(_arg(args, "seg_precision", DEFAULT_PRECISION[self.kind])))
        load_seg_model(args, model, False)                          # ImageNet init or resume
        self.model = model.float().to(self.device).train()
        self._init_training(self.model)
        self.preds = None

    def forward(self):
        self.preds = self.model.train()(ops.pad_channels(self.images, 4))

    def backward(self):
        loss = self.criterion(self.preds, self.labels)
        self.mc_G_loss = _LazyScalar(loss)
        self._backward(loss)

    def _phase(self):
        self.forward()
        self.G_solver.zero_grad()
        self.backward()

    def print_info(self, epoch, step):
        logging.info('step:{:5d} G_lr:{:.6f} G_loss:{:.5f}(mc:{:.5f})'.format(
            step, self.G_solver.param_groups[-1]['lr'], float(self.G_loss), float(self.mc_G_loss)))
