"""`NetModel` -- the reference's training-step entry point (networks/kd_model.py:27-193), H100-native underneath.

Kept surface: NetModel(args), .set_input(data), .forward(), .student_backward(), .discriminator_backward(),
.optimize_parameters(), .adjust_learning_rate(base_lr, optimizer, i_iter), .lr_poly, .print_info, .save_ckpt,
.evalute_model; attributes .student .teacher .G_solver .D_solver .preds_S .preds_T .G_loss .mc_G_loss .pi_G_loss
.pa_G_loss .D_loss (train_and_eval.py:19-30 reads them).  Ours: .at_G_loss / .mimic_G_loss (attention transfer and MIMIC, the
paper's feature-level baselines; None while off) and .mimic_adapters.

The step machinery it shares with SegModel is StepModel's (networks/step_model.py); NetModel adds the frozen teacher, the
discriminator and the distillation terms.

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

import torch
import torch.nn as nn

from .. import functions as Fn
from .. import ops
from ..utils.criterion import (CriterionAdditionalGP, CriterionAdv, CriterionAdvForG, CriterionAT, CriterionMimic,
                               CriterionPairWiseforWholeFeatAfterPool, CriterionPairWiseLocal, CriterionPixelWise, check_feature_levels,
                               check_pa_levels, check_pa_windows, feature_level_criteria, pair_wise_level_criteria)
from ..utils.utils import load_D_model, load_S_model, load_T_model
from .pspnet_combine import Conv2d
from .sagan_models import Discriminator
from .step_model import StepModel, _LazyScalar, _arg, build_seg_network

STUDENTS = ("resnet18", "espnet_c", "espnet", "mobilenetv2")

def mimic_adapters(student, teacher, levels):
    """MIMIC's 1x1 adapters (with bias, nn.Conv2d's init), one per level of check_feature_levels() with a non-zero weight, from the
    student's width at that level to the teacher's, as the two networks' level_channels() give them: key `level<ind>` for
    preds[-(ind + 1)]."""
    cs, ct = student.level_channels(), teacher.level_channels()
    return nn.ModuleDict({"level%d" % (-i - 1): Conv2d(cs[-i - 1], ct[-i - 1], 1, bias=True) for i, w in levels if w != 0.0})


class NetModel(StepModel):
    def name(self):
        return 'kd_seg'

    def __init__(self, args):
        super().__init__(args)
        # None: scalar lambda_pa / pool_scale, one pair-wise term on preds[-5]; else [(lambda, scale)] per level, level `ind` on
        # preds[-(ind + 1)] (x1, x2, x3, x4, PSP features)
        self.pa_levels = check_pa_levels(args)
        # None: every pair-wise level fully connected (the default); else (window, dilation) of the scalar term, or a list with one
        # (window or None, dilation) per level -- a window connects each pooled node to its k x k neighbours only
        self.pa_windows = check_pa_windows(args)
        # [(feat_ind, weight)]: a scalar weight is one term on preds[-5], a list one per level as for Pa
        self.at_levels = check_feature_levels(args, "lambda_at", "attention-transfer", 500.0)
        self.mimic_levels = check_feature_levels(args, "lambda_mimic", "MIMIC", 1.0)
        self.at, self.mimic = _arg(args, "at", False) == True, _arg(args, "mimic", False) == True
        self._check_device()
        self._check_kind("student", "resnet18", STUDENTS)
        device = self.device

        student = build_seg_network(self.kind, args.classes_num, args)
        load_S_model(args, student, False)                         # ImageNet init or S_resume (utils/utils.py:93-127)
        self.student = student.float().to(device).train()
        self.parallel_student = self.student

        teacher = build_seg_network("resnet101", args.classes_num)
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

        self.mimic_adapters = None
        if self.mimic:                                            # trained with the student: same flat buffer, decay, exchange, graph
            self.mimic_adapters = mimic_adapters(self.student, self.teacher, self.mimic_levels).float().to(device).train()
        self._init_training(self.student, self.D_model, extra=self.mimic_adapters)
        self.criterion_pixel_wise = CriterionPixelWise()
        if self.pa_levels is None and self.pa_windows is None:
            self.criterion_pair_wise_for_interfeat = CriterionPairWiseforWholeFeatAfterPool(scale=args.pool_scale, feat_ind=-5)
        elif self.pa_levels is None:
            window, dilation = self.pa_windows
            self.criterion_pair_wise_for_interfeat = CriterionPairWiseLocal(scale=args.pool_scale, feat_ind=-5, window=window,
                                                                            dilation=dilation)
        else:                                                     # the reference's multi-level form (kd_model.py:81)
            self.criterion_pair_wise_for_interfeat = pair_wise_level_criteria(self.pa_levels, self.pa_windows)
        self.criterion_adv = CriterionAdv(args.adv_loss_type)
        if args.adv_loss_type == 'wgan-gp':
            self.criterion_AdditionalGP = CriterionAdditionalGP(self.parallel_D, args.lambda_gp)
        self.criterion_adv_for_G = CriterionAdvForG(args.adv_loss_type)
        self.criterion_at = feature_level_criteria(self.at_levels, CriterionAT) if self.at else []
        self.criterion_mimic = feature_level_criteria(
            self.mimic_levels, lambda i: CriterionMimic(i, self.mimic_adapters["level%d" % (-i - 1)])) if self.mimic else []

        self._teacher_stream = None
        self._d_stream = None
        self.pi_G_loss = 0.0
        self.pa_G_loss = 0.0 if self.pa_levels is None else [0.0] * len(self.pa_levels)
        self.at_G_loss = self._zero_terms(self.at_levels, "lambda_at") if self.at else None
        self.mimic_G_loss = self._zero_terms(self.mimic_levels, "lambda_mimic") if self.mimic else None
        self.D_loss = 0.0

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
        preds_T[0] and the preds_T[-(ind + 1)] of every level with a non-zero weight, plus those of the weighted attention-transfer
        and MIMIC levels -- are each resized onto the grid of their own
        student counterpart (bilinear, align_corners=True; forward only, the teacher is frozen).  Equal grids (the ResNet18
        student): nothing runs.  The teacher's own logits stay in `logits_T` for the discriminator of a full-resolution student."""
        self.logits_T = self.preds_T[0]
        preds = list(self.preds_T)
        if self.pa_levels is None:
            read = (0, len(preds) - 5)
        else:
            read = [0] + ([len(preds) - 1 - ind for ind, (lam, _) in enumerate(self.pa_levels) if lam != 0.0]
                          if self.args.pa == True else [])
        read = list(read)
        for terms_on, levels in ((self.at, self.at_levels), (self.mimic, self.mimic_levels)):
            read += [len(preds) + i for i, w in levels if terms_on and w != 0.0 and len(preds) + i not in read]
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
        if self.at:
            G_loss, self.at_G_loss = self._feature_terms(G_loss, self.at_levels, self.criterion_at, "lambda_at")
        if self.mimic:
            G_loss, self.mimic_G_loss = self._feature_terms(G_loss, self.mimic_levels, self.criterion_mimic, "lambda_mimic")
        if args.ho == True:
            d_out_S = self.parallel_D(self._d_inputs()[0])
            G_loss = G_loss + args.lambda_d * self.criterion_adv_for_G(d_out_S, d_out_S)
        # the generator step only needs d D(S) / d logits: the reference's D gradients of this pass are discarded by
        # D_solver.zero_grad() (kd_model.py:154), so they are not computed
        self.D_model.skip_param_grads = True
        try:
            self._backward(G_loss)
        finally:
            self.D_model.skip_param_grads = False
            self.D_model.engine.release()

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

    def _zero_terms(self, levels, name):
        """What at_G_loss / mimic_G_loss log before the first step: 0.0, or one 0.0 per level when args.<name> is a list."""
        return [0.0] * len(levels) if isinstance(_arg(self.args, name, None), (list, tuple)) else 0.0

    def _feature_terms(self, G_loss, levels, crits, name):
        """G_loss + sum over levels of weight * term -> (that sum, the unweighted terms as lazy device scalars: a list when args.<name>
        is one, else the single term).  A level with weight 0 launches nothing and logs 0.0."""
        terms = []
        for (_, w), crit in zip(levels, crits):
            if crit is None:
                terms.append(0.0)
                continue
            temp = crit(self.preds_S, self.preds_T)
            terms.append(_LazyScalar(temp))
            G_loss = G_loss + w * temp
        return G_loss, (terms if isinstance(_arg(self.args, name, None), (list, tuple)) else terms[0])

    def _extra_states(self):
        adapters = getattr(self, "mimic_adapters", None)
        return {} if adapters is None else {"mimic_state_dict": adapters}

    def discriminator_backward(self):
        self._discriminator_phase()
        self.D_solver.all_reduce_grads(self.world)
        self.D_solver.step()

    def _phase(self):
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

    def _update(self):
        """The student's update and, with Ho, the D all-reduce + D_solver.step() (kd_model.py:171, :165)."""
        super()._update()
        if self.args.ho == True:
            self.D_solver.all_reduce_grads(self.world)
            self.D_solver.step()

    def print_info(self, epoch, step):
        def terms(v):                                               # a list: one unweighted term per level
            return '[' + ', '.join('{:.5f}'.format(float(t)) for t in v) + ']' if isinstance(v, list) else '{:.5f}'.format(float(v))
        pa = terms(self.pa_G_loss)
        for name in ('at', 'mimic'):                                # appended only while the term is on
            v = getattr(self, name + '_G_loss', None)
            if v is not None:
                pa += ' {}:{}'.format(name, terms(v))
        logging.info('step:{:5d} G_lr:{:.6f} G_loss:{:.5f}(mc:{:.5f} pixelwise:{:.5f} pairwise:{}) D_lr:{:.6f} D_loss:{:.5f}'.format(
            step, self.G_solver.param_groups[-1]['lr'], float(self.G_loss), float(self.mc_G_loss), float(self.pi_G_loss),
            pa, self.D_solver.param_groups[-1]['lr'], float(self.D_loss)))
