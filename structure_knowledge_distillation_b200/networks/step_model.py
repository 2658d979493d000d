"""`StepModel` -- the training-step machinery NetModel (distillation) and SegModel (no teacher, no discriminator) share.

Both train one network of the table below with FlatSGD (direct gradient writes) on the sm_90a kernels, one process per GPU: rank 0's
parameters are broadcast at start, the gradient is exchanged by a bucketed NCCL all-reduce issued from inside the backward pass (or,
with `allreduce='nvls'`, inside the SGD kernel), weight gradients run on a side stream, and with `cuda_graph` the step is captured
once and replayed from staged inputs.

A subclass builds its networks and defines two hooks: `_phase()`, everything a step does before the optimizer updates (what the
CUDA graph captures), and `_update()`, the updates that stay eager after it (StepModel's: the student's all-reduce and SGD step).
"""
import os
import os.path as osp

import torch
import torch.distributed as dist

from .. import functions as Fn
from ..optim import FlatSGD
from ..utils.criterion import CriterionCrossEntropy, CriterionDSN, CriterionOhemDSN, check_task_loss_weights
from .espnet import ESPNet, ESPNet_C
from .evaluate import evaluate_main
from .mobilenet import MobileNetV2
from .pspnet_combine import BasicBlock, Bottleneck, Res_pspnet

SEG_MODELS = ("resnet101", "resnet18", "espnet_c", "espnet", "mobilenetv2")


class _LazyScalar:
    """Device scalar that turns into a Python float only when somebody looks at it."""

    def __init__(self, t):
        self.t = t.detach()

    def __float__(self):
        return float(self.t)

    def __format__(self, spec):
        return format(float(self), spec)

    def __repr__(self):
        return repr(float(self))

    def item(self):
        return float(self)


def _arg(args, name, default):
    return getattr(args, name, default)


def build_seg_network(kind, classes_num, args=None):
    """The network `kind` (one of SEG_MODELS; on the CPU, parameters as constructed)."""
    if kind == "resnet101":
        return Res_pspnet(Bottleneck, [3, 4, 23, 3], num_classes=classes_num)
    if kind == "resnet18":
        return Res_pspnet(BasicBlock, [2, 2, 2, 2], num_classes=classes_num)
    if kind in ("espnet_c", "espnet"):
        return (ESPNet_C if kind == "espnet_c" else ESPNet)(classes_num, _arg(args, "espnet_p", 2), _arg(args, "espnet_q", 8))
    if kind == "mobilenetv2":
        return MobileNetV2(classes_num)
    raise ValueError("seg_model must be one of %s (got %r)" % (", ".join(repr(k) for k in SEG_MODELS), kind))


class StepModel():
    def __init__(self, args):
        """The argument checks every step model makes first; like all of its checks, before any device work."""
        self.args = args
        if not 1 <= int(args.classes_num) <= 32:              # the loss, OHEM and discriminator kernels hold up to 32 classes
            raise ValueError("classes_num must be in 1..32 (got %r)" % (args.classes_num,))
        self.class_weights = check_task_loss_weights(args)

    def _check_device(self):
        device = torch.device(_arg(self.args, "device", "cuda"))
        if device.type != "cuda":
            raise RuntimeError("%s runs on CUDA (sm_90a) only; there is no CPU path" % type(self).__name__)
        self.device = device
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1

    def _check_kind(self, option, default, kinds):
        """args.<option> names the trained network, one of `kinds`."""
        kind = str(_arg(self.args, option, default))
        if kind not in kinds:
            raise ValueError("%s must be one of %s (got %r)" % (option, ", ".join(repr(k) for k in kinds), kind))
        self.kind = kind
        # the ESPNets have no auxiliary head (single-head cross entropy) and issue their weight gradients on the main stream
        self.espnet = kind in ("espnet_c", "espnet")
        if _arg(self.args, "sync_bn", False) and (self.espnet or kind == "mobilenetv2"):
            raise ValueError("sync_bn is only available with the ResNet networks (the BatchNorm statistics of %r are per rank)" % kind)

    def _init_training(self, net, D_model=None):
        """Training state for `net` (on the device): sync_bn, FlatSGD G_solver (and D_solver for NetModel's discriminator `D_model`),
        the gradient exchange across ranks, the task criterion, the CUDA-graph option and the snapshot directory."""
        args = self.args
        if _arg(args, "sync_bn", False):                          # cross-rank batch statistics (the reference's InPlaceABNSync semantics)
            from ..libs import InPlaceABNSync
            for mod in net.modules():
                if isinstance(mod, InPlaceABNSync):
                    mod.sync_stats = True
        self._net = net

        # gradient exchange for world > 1: "nccl" = bucketed ncclAllReduce issued from inside the backward pass (default);
        # "nvls" = no NCCL on the path: the reduction happens inside the SGD kernel over NVSwitch multicast (FlatSGD.step_nvls)
        self.allreduce = str(_arg(args, "allreduce", "nccl")) if self.world > 1 else "none"
        if self.allreduce not in ("nccl", "nvls", "none"):
            raise ValueError("allreduce must be 'nccl' or 'nvls'")
        sym = self.allreduce == "nvls"
        self.G_solver = FlatSGD([p for p in net.parameters() if p.requires_grad], args.lr_g, momentum=args.momentum,
                                weight_decay=args.weight_decay, direct_grads=True, symmetric=sym)
        solvers, modules = [self.G_solver], [net]
        if D_model is not None:
            self.D_solver = FlatSGD([p for p in D_model.parameters() if p.requires_grad], args.lr_d, momentum=args.momentum,
                                    weight_decay=args.weight_decay, symmetric=sym)
            solvers.append(self.D_solver)
            modules.append(D_model)
        self.best_mean_IU = _arg(args, "best_mean_IU", 0.0)
        if self.world > 1:
            self._sync_replicas(solvers, modules)
            if sym:
                for s in solvers:
                    s.enable_nvls()
            elif int(_arg(args, "allreduce_buckets", 4)) > 0:      # 0: one all-reduce after the backward pass
                self.G_solver.enable_overlap(int(_arg(args, "allreduce_buckets", 4)))

        if _arg(args, "ohem", False):                             # OHEM task loss (the reference imports CriterionOhemDSN, kd_model.py:18)
            # (ESPNet-C: head 0 only, preds[1] is None)
            self.criterion = CriterionOhemDSN(thresh=_arg(args, "ohem_thres", 0.7), min_kept=_arg(args, "ohem_keep", 100000))
        elif self.espnet:
            self.criterion = CriterionCrossEntropy(weight=self.class_weights).to(self.device)
        else:
            self.criterion = CriterionDSN(weight=self.class_weights).to(self.device)

        self.overlap_streams = bool(_arg(args, "overlap_streams", True))
        self._graphs = None
        if _arg(args, "cuda_graph", False):
            self.enable_cuda_graphs()
        self.mc_G_loss = 0.0
        self.G_loss = 0.0
        snap = _arg(args, "snapshot_dir", None)
        if snap and not os.path.exists(snap):
            os.makedirs(snap, exist_ok=True)

    def _sync_replicas(self, solvers, modules):
        """One process per GPU: every rank starts from rank 0's parameters, BN running statistics and spectral-norm vectors (the
        reference's single-process nn.DataParallel replicates module 0 every step, utils/parallel.py:102-111; without this, layers
        that no checkpoint covers would differ per rank)."""
        for s in solvers:
            dist.broadcast(s.flat_p, 0)
        for mod in modules:
            for b in mod.buffers():
                dist.broadcast(b, 0)
            for p in mod.parameters():
                if not p.requires_grad:                             # weight_u / weight_v live outside the flat buffers
                    dist.broadcast(p.data, 0)

    # ---- the reference's step API ------------------------------------------------------------------------
    def set_input(self, data):
        images, labels = data[0], data[1]
        if self._graphs is not None and self._graphs.get("captured"):
            # replayed CUDA graphs read fixed device buffers.  The host -> device copy of the next batch goes to a STAGING pair on a
            # copy stream, so it runs while the previous step's graph is still executing (set_input returns immediately when the source
            # is pinned); optimize_parameters() moves staging -> static buffers (a 0.1 GB device copy) right before the replay.
            g = self._graphs
            if "stage_images" not in g:
                g["stage_images"], g["stage_labels"] = torch.empty_like(g["static_images"]), torch.empty_like(g["static_labels"])
                g["copy_stream"] = torch.cuda.Stream()
                g["staged"], g["consumed"] = torch.cuda.Event(), None
            cs = g["copy_stream"]
            if g["consumed"] is not None:
                cs.wait_event(g["consumed"])                          # the previous batch has left the staging buffers
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

    def _backward(self, loss):
        """loss.backward() into G_solver's flat gradient; G_loss becomes `loss`."""
        overlap = self.world > 1 and self.G_solver._buckets is not None
        if overlap:
            # bucketed NCCL all-reduce of the flat gradient, issued from inside the backward pass as each range of parameters
            # completes (utils/parallel.py:54-63,155 semantics: mean over ranks)
            self.G_solver.begin_overlapped_reduce(self.world)
        if self.overlap_streams and not self.espnet:
            # weight gradients on a side stream (the ESPNets issue theirs on the main stream: no side-stream window, so no join on
            # an idle stream, which a CUDA-graph capture would reject)
            Fn.WgradOverlap.begin()
            if Fn.WgradOverlap.stream not in self.G_solver.producer_streams:
                self.G_solver.producer_streams.append(Fn.WgradOverlap.stream)
        try:
            loss.backward()
        finally:
            Fn.WgradOverlap.end()                                 # join: weight gradients complete before the all-reduce / SGD step
            if overlap:
                self.G_solver.finish_overlapped_reduce()
        self._g_reduced = overlap
        self.G_loss = _LazyScalar(loss)

    def _update(self):
        """The all-reduce of the student gradient, unless the backward pass already did it bucket by bucket (a no-op with
        allreduce == "nvls": FlatSGD.step() reduces inside its kernel), and G_solver.step()."""
        if not getattr(self, "_g_reduced", False):
            self.G_solver.all_reduce_grads(self.world)
        self.G_solver.step()

    def optimize_parameters(self):
        if self._graphs is not None:
            return self._optimize_graphed()
        self._phase()
        self._update()

    # ---- CUDA-graph execution: the thousands of launches of a step are captured once and replayed ------------------------
    def enable_cuda_graphs(self, warmup=3):
        """Capture `_phase()` as one CUDA graph after `warmup` eager steps; `_update()` (the all-reduce when not bucketed into the
        backward pass, the SGD kernels) stays eager (the learning rate is a device scalar, so poly-LR updates need no re-capture)."""
        self._graphs = dict(calls=0, warmup=warmup, captured=False)

    def _optimize_graphed(self):
        g = self._graphs
        if not g["captured"]:
            g["calls"] += 1
            if g["calls"] <= g["warmup"]:
                # eager warm-up on a side stream (torch's CUDA-graph recipe): autograd's gradient accumulators must not be
                # bound to the legacy default stream, which cannot take part in a capture
                side = g.setdefault("side", torch.cuda.Stream())
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    self._phase()
                    self._update()
                torch.cuda.current_stream().wait_stream(side)
                return
            # static input buffers + capture
            self.images = self.images.clone(); self.labels = self.labels.clone()
            g["static_images"], g["static_labels"] = self.images, self.labels     # what the captured kernels read
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
        """evaluate_main on `model`: the eval-mode path, BN folded from the current running statistics."""
        mean_IU, IU_array = evaluate_main(model=model, loader=loader, gpu_id=gpu_id, input_size=input_size, num_classes=num_classes, whole=whole)
        return mean_IU, IU_array

    def save_ckpt(self, epoch, step, mean_IU, IU_array):
        """The trained network's state_dict to <snapshot_dir>/CS_scenes_<step>_<mean_IU>.pth -> that path.  Replicas are identical:
        rank 0 writes, other ranks return None."""
        if self.world > 1 and dist.get_rank() != 0:
            return
        path = osp.join(self.args.snapshot_dir, 'CS_scenes_' + str(step) + '_' + str(mean_IU) + '.pth')
        torch.save(self._net.state_dict(), path)
        return path
