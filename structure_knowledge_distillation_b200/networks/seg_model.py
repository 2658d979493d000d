"""`SegModel` -- a segmentation training step with no teacher and no discriminator, on the same sm_90a kernels as NetModel's student.

It trains what NetModel distills from: the PSPNet-ResNet101 teacher (`seg_model='resnet101'`, the default), for a class count or a crop
size nobody publishes a checkpoint for, and every student kind without distillation (the reference's "baseline" row: ResNet18-PSP
trained on the task loss alone).  The step API is NetModel's (set_input, forward, backward, optimize_parameters, adjust_learning_rate,
lr_poly, print_info, save_ckpt, evalute_model; .model .G_solver .preds .G_loss .mc_G_loss), so a train_and_eval.py-style loop drives
it unchanged, and what save_ckpt writes loads through load_T_model as NetModel's teacher (`T_ckpt_path`).

Underneath, as for NetModel's student: FlatSGD with direct gradient writes, weight gradients on a side stream, one process per GPU with
rank 0's parameters broadcast at start and the bucketed NCCL all-reduce (or `allreduce='nvls'`), `sync_bn` for the ResNets, and the
`cuda_graph` option with staged inputs.
"""
import logging
import os
import os.path as osp

import torch
import torch.distributed as dist

from .. import functions as Fn
from .. import ops
from ..optim import FlatSGD
from ..utils.criterion import CriterionCrossEntropy, CriterionDSN, CriterionOhemDSN
from ..utils.utils import load_seg_model
from .espnet import ESPNet, ESPNet_C
from .evaluate import evaluate_main
from .kd_model import _LazyScalar, _arg
from .mobilenet import MobileNetV2
from .pspnet_combine import BasicBlock, Bottleneck, Conv2d, Res_pspnet

SEG_MODELS = ("resnet101", "resnet18", "espnet_c", "espnet", "mobilenetv2")

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


def build_seg_network(kind, classes_num, args=None):
    """The network `seg_model=kind` trains (on the CPU, parameters as constructed)."""
    if kind == "resnet101":
        return Res_pspnet(Bottleneck, [3, 4, 23, 3], num_classes=classes_num)
    if kind == "resnet18":
        return Res_pspnet(BasicBlock, [2, 2, 2, 2], num_classes=classes_num)
    if kind in ("espnet_c", "espnet"):
        return (ESPNet_C if kind == "espnet_c" else ESPNet)(classes_num, _arg(args, "espnet_p", 2), _arg(args, "espnet_q", 8))
    if kind == "mobilenetv2":
        return MobileNetV2(classes_num)
    raise ValueError("seg_model must be one of %s (got %r)" % (", ".join(repr(k) for k in SEG_MODELS), kind))


class SegModel():
    def name(self):
        return 'seg'

    def __init__(self, args):
        self.args = args
        if not 1 <= int(args.classes_num) <= 32:              # the loss and OHEM kernels hold up to 32 classes
            raise ValueError("classes_num must be in 1..32 (got %r)" % (args.classes_num,))
        self.kind = str(_arg(args, "seg_model", "resnet101"))
        if self.kind not in SEG_MODELS:
            raise ValueError("seg_model must be one of %s (got %r)" % (", ".join(repr(k) for k in SEG_MODELS), self.kind))
        sync_bn = bool(_arg(args, "sync_bn", False))
        if sync_bn and self.kind not in ("resnet101", "resnet18"):
            raise ValueError("sync_bn is only available with the ResNet networks (the BatchNorm statistics of %r are per rank)" % self.kind)
        device = torch.device(_arg(args, "device", "cuda"))
        if device.type != "cuda":
            raise RuntimeError("SegModel runs on CUDA (sm_90a) only; there is no CPU path")
        self.device = device
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1

        model = build_seg_network(self.kind, args.classes_num, args)
        if self.kind in DEFAULT_PRECISION:
            set_precision_policy(model, str(_arg(args, "seg_precision", DEFAULT_PRECISION[self.kind])))
        load_seg_model(args, model, False)                          # ImageNet init or resume
        self.model = model.float().to(device).train()
        if sync_bn:                                                 # cross-rank batch statistics (InPlaceABNSync semantics)
            from ..libs import InPlaceABNSync
            for mod in self.model.modules():
                if isinstance(mod, InPlaceABNSync):
                    mod.sync_stats = True

        self.allreduce = str(_arg(args, "allreduce", "nccl")) if self.world > 1 else "none"
        if self.allreduce not in ("nccl", "nvls", "none"):
            raise ValueError("allreduce must be 'nccl' or 'nvls'")
        sym = self.allreduce == "nvls"
        self.G_solver = FlatSGD([p for p in self.model.parameters() if p.requires_grad], args.lr_g, momentum=args.momentum,
                                weight_decay=args.weight_decay, direct_grads=True, symmetric=sym)
        self.best_mean_IU = _arg(args, "best_mean_IU", 0.0)
        if self.world > 1:
            self._sync_replicas()
            if sym:
                self.G_solver.enable_nvls()
            elif int(_arg(args, "allreduce_buckets", 4)) > 0:      # 0: one all-reduce after the backward pass
                self.G_solver.enable_overlap(int(_arg(args, "allreduce_buckets", 4)))

        if _arg(args, "ohem", False):
            self.criterion = CriterionOhemDSN(thresh=_arg(args, "ohem_thres", 0.7), min_kept=_arg(args, "ohem_keep", 100000))
        elif self.kind in ("espnet_c", "espnet"):                   # no auxiliary head
            self.criterion = CriterionCrossEntropy()
        else:
            self.criterion = CriterionDSN()

        self.overlap_streams = bool(_arg(args, "overlap_streams", True))
        self._graphs = None
        if _arg(args, "cuda_graph", False):
            self.enable_cuda_graphs()
        self.preds = None
        self.mc_G_loss = 0.0
        self.G_loss = 0.0
        snap = _arg(args, "snapshot_dir", None)
        if snap and not os.path.exists(snap):
            os.makedirs(snap, exist_ok=True)

    def _sync_replicas(self):
        """Every rank starts from rank 0's parameters and BN running statistics (NetModel._sync_replicas)."""
        dist.broadcast(self.G_solver.flat_p, 0)
        for b in self.model.buffers():
            dist.broadcast(b, 0)

    # ---- the step API ------------------------------------------------------------------------------------
    def set_input(self, data):
        images, labels = data[0], data[1]
        if self._graphs is not None and self._graphs.get("captured"):
            # replayed CUDA graph: the next batch goes to a staging pair on a copy stream (NetModel.set_input)
            g = self._graphs
            if "stage_images" not in g:
                g["stage_images"], g["stage_labels"] = torch.empty_like(g["static_images"]), torch.empty_like(g["static_labels"])
                g["copy_stream"] = torch.cuda.Stream()
                g["staged"], g["consumed"] = torch.cuda.Event(), None
            cs = g["copy_stream"]
            if g["consumed"] is not None:
                cs.wait_event(g["consumed"])
            with torch.cuda.stream(cs):
                g["stage_images"].copy_(images, non_blocking=True)
                g["stage_labels"].copy_(labels, non_blocking=True)
                g["staged"].record(cs)
            g["pending"] = True
            return
        self.images = images.to(self.device, non_blocking=True)
        self.labels = labels.long().to(self.device, non_blocking=True)

    def lr_poly(self, base_lr, iter, max_iter, power):
        return base_lr * ((1 - float(iter) / max_iter) ** (power))

    def adjust_learning_rate(self, base_lr, optimizer, i_iter):
        lr = self.lr_poly(base_lr, i_iter, self.args.num_steps, self.args.power)
        optimizer.param_groups[0]['lr'] = lr
        return lr

    def forward(self):
        self.preds = self.model.train()(ops.pad_channels(self.images, 4))

    def backward(self):
        loss = self.criterion(self.preds, self.labels)
        self.mc_G_loss = _LazyScalar(loss)
        overlap = self.world > 1 and self.G_solver._buckets is not None
        if overlap:                                                 # bucketed all-reduce issued from inside the backward pass
            self.G_solver.begin_overlapped_reduce(self.world)
        if self.overlap_streams and self.kind in ("resnet101", "resnet18", "mobilenetv2"):
            Fn.WgradOverlap.begin()                                 # weight gradients on the side stream
            if Fn.WgradOverlap.stream not in self.G_solver.producer_streams:
                self.G_solver.producer_streams.append(Fn.WgradOverlap.stream)
        try:
            loss.backward()
        finally:
            Fn.WgradOverlap.end()
            if overlap:
                self.G_solver.finish_overlapped_reduce()
        self._g_reduced = overlap
        self.G_loss = _LazyScalar(loss)

    def _phase(self):
        self.forward()
        self.G_solver.zero_grad()
        self.backward()

    def _update(self):
        if not getattr(self, "_g_reduced", False):
            self.G_solver.all_reduce_grads(self.world)              # no-op with allreduce == "nvls": step() reduces in its kernel
        self.G_solver.step()

    def optimize_parameters(self):
        if self._graphs is not None:
            return self._optimize_graphed()
        self._phase()
        self._update()

    # ---- CUDA-graph execution ------------------------------------------------------------------------------
    def enable_cuda_graphs(self, warmup=3):
        """Capture forward, loss and backward as one CUDA graph after `warmup` eager steps; the all-reduce (when not bucketed into the
        backward) and the SGD kernel stay eager (the learning rate is a device scalar, so poly-LR updates need no re-capture)."""
        self._graphs = dict(calls=0, warmup=warmup, captured=False)

    def _optimize_graphed(self):
        g = self._graphs
        if not g["captured"]:
            g["calls"] += 1
            if g["calls"] <= g["warmup"]:
                side = g.setdefault("side", torch.cuda.Stream())    # eager warm-up off the legacy default stream
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    self._phase()
                    self._update()
                torch.cuda.current_stream().wait_stream(side)
                return
            self.images = self.images.clone(); self.labels = self.labels.clone()
            g["static_images"], g["static_labels"] = self.images, self.labels
            torch.cuda.synchronize()
            g["graph"] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g["graph"]):
                self._phase()
            self._update()
            g["captured"] = True
            return
        if g.get("pending"):                                        # staged batch -> the graph's static input buffers
            cur = torch.cuda.current_stream()
            cur.wait_event(g["staged"])
            g["static_images"].copy_(g["stage_images"], non_blocking=True)
            g["static_labels"].copy_(g["stage_labels"], non_blocking=True)
            self.images, self.labels = g["static_images"], g["static_labels"]
            g["consumed"] = torch.cuda.Event(); g["consumed"].record(cur)
            g["pending"] = False
        g["graph"].replay()
        self._update()

    def evalute_model(self, model, loader, gpu_id, input_size, num_classes, whole):
        """evaluate_main on `model` (normally self.model): the eval-mode path, BN folded from the current running statistics."""
        mean_IU, IU_array = evaluate_main(model=model, loader=loader, gpu_id=gpu_id, input_size=input_size, num_classes=num_classes, whole=whole)
        return mean_IU, IU_array

    def print_info(self, epoch, step):
        logging.info('step:{:5d} G_lr:{:.6f} G_loss:{:.5f}(mc:{:.5f})'.format(
            step, self.G_solver.param_groups[-1]['lr'], float(self.G_loss), float(self.mc_G_loss)))

    def save_ckpt(self, epoch, step, mean_IU, IU_array):
        """model.state_dict() under the Res_pspnet names (loadable as NetModel's teacher through load_T_model); rank 0 writes."""
        if self.world > 1 and dist.get_rank() != 0:
            return
        path = osp.join(self.args.snapshot_dir, 'CS_scenes_' + str(step) + '_' + str(mean_IU) + '.pth')
        torch.save(self.model.state_dict(), path)
        return path
