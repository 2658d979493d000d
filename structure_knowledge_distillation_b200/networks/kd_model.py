"""`NetModel` -- the reference's training-step entry point (networks/kd_model.py:27-193), H100-native underneath.

Kept surface: NetModel(args), .set_input(data), .forward(), .student_backward(), .discriminator_backward(),
.optimize_parameters(), .adjust_learning_rate(base_lr, optimizer, i_iter), .lr_poly, .print_info, .save_ckpt,
.evalute_model; attributes .student .teacher .G_solver .D_solver .preds_S .preds_T .G_loss .mc_G_loss .pi_G_loss
.pa_G_loss .D_loss (train_and_eval.py:19-30 reads them).

What changed underneath (DESIGN.md):
  * single-process nn.DataParallel replicas + per-step parameter broadcast (utils/parallel.py) -> one process per GPU,
    persistent replicas, ONE NCCL all-reduce (mean) of the flat student-gradient buffer per step (+ one for D when Ho);
    per-rank loss on the local shard and averaged gradients == the reference's mean-over-GPUs semantics
    (utils/parallel.py:155);
  * scalar logging is lazy: the five `.item()` host syncs per step (kd_model.py:130-164) become device scalars that are
    only read when print_info()/the attribute is used;
  * the discarded teacher cross-entropy (kd_model.py:129) is not computed.
"""
import logging
import os
import os.path as osp

import torch
import torch.distributed as dist

from .. import functions as Fn
from .. import ops
from ..optim import FlatSGD
from ..utils.criterion import (CriterionAdditionalGP, CriterionAdv, CriterionAdvForG, CriterionCrossEntropy, CriterionDSN,
                               CriterionOhemDSN, CriterionPairWiseforWholeFeatAfterPool, CriterionPixelWise,
                               check_pa_levels, check_task_loss_weights, pair_wise_level_criteria)
from ..utils.utils import load_D_model, load_S_model, load_T_model
from .espnet import ESPNet, ESPNet_C
from .evaluate import evaluate_main
from .mobilenet import MobileNetV2
from .pspnet_combine import BasicBlock, Bottleneck, Res_pspnet
from .sagan_models import Discriminator


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


class NetModel():
    def name(self):
        return 'kd_seg'

    def __init__(self, args):
        self.args = args
        if not 1 <= int(args.classes_num) <= 32:              # the loss, OHEM and discriminator kernels hold up to 32 classes
            raise ValueError("classes_num must be in 1..32 (got %r)" % (args.classes_num,))
        class_weights = check_task_loss_weights(args)
        # None: scalar lambda_pa / pool_scale, one pair-wise term on preds[-5]; else [(lambda, scale)] per level, level `ind` on
        # preds[-(ind + 1)] (x1, x2, x3, x4, PSP features)
        self.pa_levels = check_pa_levels(args)
        device = torch.device(_arg(args, "device", "cuda"))
        if device.type != "cuda":
            raise RuntimeError("NetModel runs on CUDA (sm_90a) only; there is no CPU path")
        self.device = device
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1

        self.student_kind = str(_arg(args, "student", "resnet18"))
        if self.student_kind == "resnet18":
            student = Res_pspnet(BasicBlock, [2, 2, 2, 2], num_classes=args.classes_num)
        elif self.student_kind in ("espnet_c", "espnet"):
            if _arg(args, "sync_bn", False):
                raise ValueError("sync_bn is not available with the ESPNet students (their BatchNorm statistics are per rank)")
            student = (ESPNet_C if self.student_kind == "espnet_c" else ESPNet)(args.classes_num, _arg(args, "espnet_p", 2),
                                                                               _arg(args, "espnet_q", 8))
        elif self.student_kind == "mobilenetv2":
            if _arg(args, "sync_bn", False):
                raise ValueError("sync_bn is not available with the MobileNetV2 student (its BatchNorm statistics are per rank)")
            student = MobileNetV2(args.classes_num)
        else:
            raise ValueError("student must be 'resnet18', 'espnet_c', 'espnet' or 'mobilenetv2' (got %r)" % self.student_kind)
        load_S_model(args, student, False)                         # ImageNet init or S_resume (utils/utils.py:93-127)
        self.student = student.float().to(device).train()
        if _arg(args, "sync_bn", False):                          # cross-rank batch statistics (the reference's InPlaceABNSync semantics)
            from ..libs import InPlaceABNSync
            for mod in self.student.modules():
                if isinstance(mod, InPlaceABNSync):
                    mod.sync_stats = True
        self.parallel_student = self.student

        teacher = Res_pspnet(Bottleneck, [3, 4, 23, 3], num_classes=args.classes_num)
        load_T_model(teacher, _arg(args, "T_ckpt_path", None))
        self.teacher = teacher.float().to(device).eval()
        for p in self.teacher.parameters():
            p.requires_grad_(False)
        self.parallel_teacher = self.teacher

        # SAGAN discriminator on the sm_90a kernels (networks/sagan_engine.py): wgmma spectral-norm convolutions, fused
        # attention, and the WGAN-GP penalty by a tangent + joint reverse pass instead of autograd's double backward
        D_model = Discriminator(args.preprocess_GAN_mode, args.classes_num, args.batch_size, args.imsize_for_adv, args.adv_conv_dim)
        load_D_model(args, D_model, False)
        self.D_model = D_model.float().to(device).train()
        self.parallel_D = self.D_model

        # gradient exchange for world > 1: "nccl" = bucketed ncclAllReduce issued from inside the backward pass (default);
        # "nvls" = no NCCL on the path: the reduction happens inside the SGD kernel over NVSwitch multicast (FlatSGD.step_nvls)
        self.allreduce = str(_arg(args, "allreduce", "nccl")) if self.world > 1 else "none"
        if self.allreduce not in ("nccl", "nvls", "none"):
            raise ValueError("allreduce must be 'nccl' or 'nvls'")
        sym = self.allreduce == "nvls"
        self.G_solver = FlatSGD([p for p in self.student.parameters() if p.requires_grad], args.lr_g, momentum=args.momentum,
                                weight_decay=args.weight_decay, direct_grads=True, symmetric=sym)
        self.D_solver = FlatSGD([p for p in self.D_model.parameters() if p.requires_grad], args.lr_d, momentum=args.momentum,
                                weight_decay=args.weight_decay, symmetric=sym)
        self.best_mean_IU = _arg(args, "best_mean_IU", 0.0)
        if self.world > 1:
            self._sync_replicas()
            if sym:
                self.G_solver.enable_nvls()
                self.D_solver.enable_nvls()
            elif int(_arg(args, "allreduce_buckets", 4)) > 0:      # 0: one all-reduce after the backward pass
                self.G_solver.enable_overlap(int(_arg(args, "allreduce_buckets", 4)))

        if _arg(args, "ohem", False):                             # OHEM task loss (the reference imports CriterionOhemDSN, kd_model.py:18)
            # (ESPNet-C: head 0 only, preds[1] is None)
            self.criterion = CriterionOhemDSN(thresh=_arg(args, "ohem_thres", 0.7), min_kept=_arg(args, "ohem_keep", 100000))
        elif self.student_kind in ("espnet_c", "espnet"):         # the ESPNets: no auxiliary head, single-head cross entropy
            self.criterion = CriterionCrossEntropy(weight=class_weights).to(device)
        else:
            self.criterion = CriterionDSN(weight=class_weights).to(device)
        self.criterion_pixel_wise = CriterionPixelWise()
        if self.pa_levels is None:
            self.criterion_pair_wise_for_interfeat = CriterionPairWiseforWholeFeatAfterPool(scale=args.pool_scale, feat_ind=-5)
        else:                                                     # the reference's multi-level form (kd_model.py:81)
            self.criterion_pair_wise_for_interfeat = pair_wise_level_criteria(self.pa_levels)
        self.criterion_adv = CriterionAdv(args.adv_loss_type)
        if args.adv_loss_type == 'wgan-gp':
            self.criterion_AdditionalGP = CriterionAdditionalGP(self.parallel_D, args.lambda_gp)
        self.criterion_adv_for_G = CriterionAdvForG(args.adv_loss_type)

        self.overlap_streams = bool(_arg(args, "overlap_streams", True))
        self._teacher_stream = None
        self._d_stream = None
        self._graphs = None
        if _arg(args, "cuda_graph", False):
            self.enable_cuda_graphs()
        self.mc_G_loss = 0.0
        self.pi_G_loss = 0.0
        self.pa_G_loss = 0.0 if self.pa_levels is None else [0.0] * len(self.pa_levels)
        self.D_loss = 0.0
        self.G_loss = 0.0
        snap = _arg(args, "snapshot_dir", None)
        if snap and not os.path.exists(snap):
            os.makedirs(snap, exist_ok=True)

    def _sync_replicas(self):
        """One process per GPU: every rank starts from rank 0's student / discriminator parameters, BN running statistics and
        spectral-norm vectors (the reference's single-process nn.DataParallel replicates module 0 every step,
        utils/parallel.py:102-111; without this, layers that no checkpoint covers would differ per rank)."""
        dist.broadcast(self.G_solver.flat_p, 0)
        dist.broadcast(self.D_solver.flat_p, 0)
        for mod in (self.student, self.D_model):
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

    def forward(self):
        images = ops.pad_channels(self.images, 4)                 # shared by teacher and student
        if not self.overlap_streams:
            with torch.no_grad():
                self.preds_T = self.parallel_teacher.eval()(images)
            self.preds_S = self.parallel_student.train()(images)
            self._resample_teacher()
            return
        # the frozen teacher and the student are independent until the losses: the teacher's forward goes to a second stream, so the
        # student's HBM-bound passes (ABN statistics / apply, pooling) run under the teacher's tensor-bound convolutions (one
        # persistent conv CTA per SM leaves registers for one elementwise CTA beside it) instead of between them
        cur = torch.cuda.current_stream()
        if self._teacher_stream is None:
            self._teacher_stream = torch.cuda.Stream()
        side = self._teacher_stream
        side.wait_stream(cur)
        with torch.cuda.stream(side), torch.no_grad():
            self.preds_T = self.parallel_teacher.eval()(images)
        self.preds_S = self.parallel_student.train()(images)
        cur.wait_stream(side)
        self._resample_teacher()

    def _resample_teacher(self):
        """Students on another grid than the teacher (ESPNet-C: 45x60 at 360x480, PSPNet's ceil-mode pool: 46x61; the full ESPNet's
        logits: 360x480): the teacher tensors the distillation terms read -- preds_T[0] and preds_T[-5], or with pair-wise levels
        preds_T[0] and the preds_T[-(ind + 1)] of every level with a non-zero weight -- are each resized onto the grid of their own
        student counterpart (bilinear, align_corners=True; forward only, the teacher is frozen).  Equal grids (the ResNet18
        student): nothing runs.  The teacher's own logits stay in `logits_T` for the discriminator of a full-resolution student."""
        self.logits_T = self.preds_T[0]
        preds = list(self.preds_T)
        if self.pa_levels is None:
            read = (0, len(preds) - 5)
        else:
            read = [0] + ([len(preds) - 1 - ind for ind, (lam, _) in enumerate(self.pa_levels) if lam != 0.0]
                          if self.args.pa == True else [])
        for i in read:
            size = tuple(self.preds_S[i].shape[2:])
            if tuple(preds[i].shape[2:]) != size:
                preds[i] = ops.resample_nhwc(preds[i], *size)
        self.preds_T = preds

    def _d_inputs(self):
        """-> (student, teacher) logits the discriminator sees.  A student whose logits are at the input resolution (the full ESPNet)
        meets D on the teacher's logit grid: its logits resized onto that grid (bilinear, align_corners=True, with the gradient of
        Fn.ResampleBilinear) against the teacher's logits as they came out.  Others: preds_S[0] against preds_T[0]."""
        s = self.preds_S[0]
        if tuple(s.shape[2:]) != tuple(self.images.shape[2:]):
            return s, self.preds_T[0]
        t = self.logits_T
        return Fn.ResampleBilinear.apply(s, t.shape[2], t.shape[3]), t

    def student_backward(self):
        args = self.args
        temp = self.criterion(self.preds_S, self.labels)
        self.mc_G_loss = _LazyScalar(temp)
        G_loss = temp
        if args.pi == True:
            temp = args.lambda_pi * self.criterion_pixel_wise(self.preds_S, self.preds_T)
            self.pi_G_loss = _LazyScalar(temp)
            G_loss = G_loss + temp
        if args.pa == True and self.pa_levels is not None:
            G_loss = self._pa_levels_loss(G_loss)
        elif args.pa == True:
            temp1 = self.criterion_pair_wise_for_interfeat(self.preds_S, self.preds_T)
            self.pa_G_loss = _LazyScalar(temp1)
            G_loss = G_loss + args.lambda_pa * temp1
        if args.ho == True:
            d_out_S = self.parallel_D(self._d_inputs()[0])
            G_loss = G_loss + args.lambda_d * self.criterion_adv_for_G(d_out_S, d_out_S)
        # the generator step only needs d D(S) / d logits: the reference's D gradients of this pass are discarded by
        # D_solver.zero_grad() (kd_model.py:154), so they are not computed
        self.D_model.skip_param_grads = True
        overlap = self.world > 1 and self.G_solver._buckets is not None
        if overlap:
            # the ONE collective of the path (teacher frozen): bucketed NCCL all-reduce of the flat student gradient, issued from
            # inside the backward pass as each range of parameters completes (utils/parallel.py:54-63,155 semantics: mean over ranks)
            self.G_solver.begin_overlapped_reduce(self.world)
        if self.overlap_streams and self.student_kind in ("resnet18", "mobilenetv2"):
            # (ESPNet-C issues its weight gradients on the main stream: no side-stream window, so no join on an idle stream, which
            # a CUDA-graph capture would reject)
            Fn.WgradOverlap.begin()
            if Fn.WgradOverlap.stream not in self.G_solver.producer_streams:
                self.G_solver.producer_streams.append(Fn.WgradOverlap.stream)
        try:
            G_loss.backward()
        finally:
            Fn.WgradOverlap.end()                                 # join: weight gradients complete before the all-reduce / SGD step
            self.D_model.skip_param_grads = False
            self.D_model.engine.release()
            if overlap:
                self.G_solver.finish_overlapped_reduce()
        self._g_reduced = overlap
        self.G_loss = _LazyScalar(G_loss)

    def _pa_levels_loss(self, G_loss):
        """G_loss + sum over levels of lambda_pa[ind] * Pa(preds[-(ind + 1)]) (kd_model.py:137-143).  A level with lambda 0 launches
        nothing and logs 0.0; pa_G_loss holds each level's unweighted term as a lazy device scalar."""
        pa = []
        for ind, ((lam, scale), crit) in enumerate(zip(self.pa_levels, self.criterion_pair_wise_for_interfeat)):
            if lam == 0.0:
                pa.append(0.0)
                continue
            h, w = self.preds_T[crit.feat_ind].shape[2:]
            if int(h * scale) < 1 or int(w * scale) < 1:
                raise ValueError("pair-wise level %d (preds[%d], %dx%d): pool_scale %r gives a %dx%d pooling window; raise the "
                                 "scale or the input size" % (ind, crit.feat_ind, h, w, scale, int(h * scale), int(w * scale)))
            temp = crit(self.preds_S, self.preds_T)
            pa.append(_LazyScalar(temp))
            G_loss = G_loss + lam * temp
        self.pa_G_loss = pa
        return G_loss

    def discriminator_backward(self):
        self._discriminator_phase()
        self.D_solver.all_reduce_grads(self.world)
        self.D_solver.step()

    def _student_and_discriminator_phases(self):
        """One step up to (not including) the two optimizer updates, with the discriminator phase (kd_model.py:153-163 without the
        D step) on its own stream UNDER the student's backward pass.  The D phase needs the logits of forward() and the D state left
        by the generator pass's D(S) (one power iteration) -- not the student's gradients or its updated weights -- and its ~370
        launches are tiny grids (4x8 .. 32x64 maps): alone they leave the GPU mostly idle, beside the student's
        backward kernels they cost nothing.  It starts once the generator pass's adjoint through D has been issued (event recorded
        by DiscriminatorFn.backward) and is joined before the optimizer updates."""
        self.forward()
        self.G_solver.zero_grad()
        if not (self.args.ho == True and self.overlap_streams):
            self.student_backward()
            if self.args.ho == True:
                self._discriminator_phase()
            return
        if self._d_stream is None:
            self._d_stream = torch.cuda.Stream()
        ev = torch.cuda.Event()
        self.D_model.adjoint_done_event = ev
        try:
            self.student_backward()                        # enqueues the whole backward; the event sits right after D's adjoint
        finally:
            self.D_model.adjoint_done_event = None
        cur = torch.cuda.current_stream()
        self._d_stream.wait_event(ev)
        with torch.cuda.stream(self._d_stream):
            self._discriminator_phase()
        cur.wait_stream(self._d_stream)

    def _reduce_G(self):
        """all-reduce of the student gradient unless the backward pass already did it bucket by bucket"""
        if not getattr(self, "_g_reduced", False):
            self.G_solver.all_reduce_grads(self.world)

    def _student_phase(self):
        self.forward()
        self.G_solver.zero_grad()
        self.student_backward()

    def _discriminator_phase(self):
        """discriminator_backward() without the optimizer step (kd_model.py:153-163)."""
        self.D_solver.zero_grad()
        args = self.args
        D = self.D_model
        D.engine.prepare()                                   # weights are constant within the phase: stage them once
        D.accumulate_into_grad = True                        # the three passes add straight into FlatSGD's gradient buffer
        try:
            with torch.no_grad():
                d_in_S, d_in_T = self._d_inputs()
            d_out_T = self.parallel_D(d_in_T.detach())
            d_out_S = self.parallel_D(d_in_S.detach())
            d_loss = args.lambda_d * self.criterion_adv(d_out_S, d_out_T)
            if args.adv_loss_type == 'wgan-gp':
                d_loss = d_loss + args.lambda_d * self.criterion_AdditionalGP([d_in_S], [d_in_T])
            d_loss.backward()
        finally:
            D.accumulate_into_grad = False
            D.engine.release()
        self.D_loss = _LazyScalar(d_loss)

    def _updates(self):
        """G_solver.step() and, with Ho, the D all-reduce + D_solver.step() (kd_model.py:171, :165)."""
        self._reduce_G()                                     # no-ops with allreduce == "nvls": FlatSGD.step() reduces inside its kernel
        self.G_solver.step()
        if self.args.ho == True:
            self.D_solver.all_reduce_grads(self.world)
            self.D_solver.step()

    def optimize_parameters(self):
        if self._graphs is not None:
            return self._optimize_graphed()
        self._student_and_discriminator_phases()
        self._updates()

    # ---- CUDA-graph execution: the ~4 000 launches of a step are captured once and replayed ------------------------
    def enable_cuda_graphs(self, warmup=3):
        """Capture the student phase (teacher fwd, student fwd, losses, backward) and the discriminator phase as two CUDA
        graphs after `warmup` eager steps; the NCCL all-reduce and the two fused SGD kernels stay eager between them
        (the learning rate is a device scalar, so poly-LR updates need no re-capture)."""
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
                    self._student_and_discriminator_phases()
                    self._updates()
                torch.cuda.current_stream().wait_stream(side)
                return
            # static input buffers + capture
            self.images = self.images.clone(); self.labels = self.labels.clone()
            g["static_images"], g["static_labels"] = self.images, self.labels     # what the captured kernels read
            torch.cuda.synchronize()
            g["student"] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g["student"]):
                self._student_and_discriminator_phases()     # ONE graph: teacher || student forward, backward || wgrad || D phase
            self._updates()
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
        g["student"].replay()
        self._updates()

    def evalute_model(self, model, loader, gpu_id, input_size, num_classes, whole):
        mean_IU, IU_array = evaluate_main(model=model, loader=loader, gpu_id=gpu_id, input_size=input_size, num_classes=num_classes, whole=whole)
        return mean_IU, IU_array

    def print_info(self, epoch, step):
        if isinstance(self.pa_G_loss, list):                        # one unweighted term per pair-wise level
            pa = '[' + ', '.join('{:.5f}'.format(float(v)) for v in self.pa_G_loss) + ']'
        else:
            pa = '{:.5f}'.format(float(self.pa_G_loss))
        logging.info('step:{:5d} G_lr:{:.6f} G_loss:{:.5f}(mc:{:.5f} pixelwise:{:.5f} pairwise:{}) D_lr:{:.6f} D_loss:{:.5f}'.format(
            step, self.G_solver.param_groups[-1]['lr'], float(self.G_loss), float(self.mc_G_loss), float(self.pi_G_loss),
            pa, self.D_solver.param_groups[-1]['lr'], float(self.D_loss)))

    def save_ckpt(self, epoch, step, mean_IU, IU_array):
        if self.world > 1 and dist.get_rank() != 0:
            return                                                  # replicas are identical: rank 0 writes
        torch.save(self.student.state_dict(), osp.join(self.args.snapshot_dir, 'CS_scenes_' + str(step) + '_' + str(mean_IU) + '.pth'))
