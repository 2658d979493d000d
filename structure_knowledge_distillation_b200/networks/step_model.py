"""`StepModel` -- the training-step machinery NetModel (distillation) and SegModel (no teacher, no discriminator) share.

Both train one network of the table below with FlatSGD (direct gradient writes) on the sm_90a kernels, one process per GPU: rank 0's
parameters are broadcast at start, the gradient is exchanged by a bucketed NCCL all-reduce issued from inside the backward pass (or,
with `allreduce='nvls'`, inside the SGD kernel), weight gradients run on a side stream, and with `cuda_graph` the step is captured
once and replayed from staged inputs.

A subclass builds its networks and defines two hooks: `_phase()`, everything a step does before the optimizer updates (what the
CUDA graph captures), and `_update()`, the updates that stay eager after it (StepModel's: the student's all-reduce and SGD step).

`save_training_state` / `load_training_state` write and restore everything a run needs to continue where it stopped (DESIGN.md §8).
"""
import os
import os.path as osp
import random
import tempfile

import numpy as np
import torch
import torch.distributed as dist

from .. import functions as Fn
from ..optim import FlatSGD
from ..utils.criterion import CriterionCrossEntropy, CriterionDSN, CriterionOhemDSN, check_task_loss_weights
from ..utils.utils import _torch_load
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


TRAINING_STATE_FORMAT = "skd-training-state"
TRAINING_STATE_VERSION = 1


def _cpu_state(module):
    return {k: v.detach().cpu().clone() for k, v in module.state_dict().items()}


def _check_state_dict(field, have, saved):
    """ValueError naming `field` unless `saved` has exactly the keys and shapes of the module state dict `have`."""
    if not isinstance(saved, dict) or set(saved) != set(have):
        missing, extra = sorted(set(have) - set(saved or ())), sorted(set(saved or ()) - set(have))
        raise ValueError("training state does not match the model: %s keys differ (missing %s, unexpected %s)"
                         % (field, missing[:5], extra[:5]))
    for k, v in have.items():
        if tuple(saved[k].shape) != tuple(v.shape):
            raise ValueError("training state does not match the model: %s[%r] has shape %s, the model's %s"
                             % (field, k, tuple(saved[k].shape), tuple(v.shape)))


def _rng_states(device, loader):
    """This process's random streams: torch CPU, the CUDA generator of `device`, Python `random`, numpy's global generator (as plain
    values, so the file loads with weights_only=True), and `loader`'s position."""
    name, keys, pos, has_gauss, gauss = np.random.get_state()
    return dict(torch=torch.get_rng_state(), cuda=torch.cuda.get_rng_state(device) if device.type == "cuda" else None,
                random=random.getstate(), numpy=(name, torch.from_numpy(keys.astype(np.int64)), int(pos), int(has_gauss), float(gauss)),
                loader=None if loader is None else loader.state_dict())


def _set_rng_states(st, device):
    torch.set_rng_state(st["torch"])
    if st["cuda"] is not None and device.type == "cuda":
        # sets the generator's seed and Philox offset in place: a captured CUDA graph reads both from the generator at every replay
        torch.cuda.set_rng_state(st["cuda"], device)
    random.setstate(st["random"])
    name, keys, pos, has_gauss, gauss = st["numpy"]
    np.random.set_state((name, keys.numpy().astype(np.uint32), pos, has_gauss, gauss))


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
        self.kind, self.kind_option = kind, option
        # the ESPNets have no auxiliary head (single-head cross entropy) and issue their weight gradients on the main stream
        self.espnet = kind in ("espnet_c", "espnet")
        if _arg(self.args, "sync_bn", False) and (self.espnet or kind == "mobilenetv2"):
            raise ValueError("sync_bn is only available with the ResNet networks (the BatchNorm statistics of %r are per rank)" % kind)

    def _init_training(self, net, D_model=None, extra=None):
        """Training state for `net` (on the device): sync_bn, FlatSGD G_solver (and D_solver for NetModel's discriminator `D_model`),
        the gradient exchange across ranks, the task criterion, the CUDA-graph option and the snapshot directory.  `extra`: a module
        trained with `net` (NetModel's MIMIC and CWD adapters), its parameters after net's in G_solver's flat buffer."""
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
        trained = list(net.parameters()) + (list(extra.parameters()) if extra is not None else [])
        self.G_solver = FlatSGD([p for p in trained if p.requires_grad], args.lr_g, momentum=args.momentum,
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

    def evalute_model(self, model, loader, gpu_id, input_size, num_classes, whole, distributed=False):
        """evaluate_main on `model`: the eval-mode path, BN folded from the current running statistics.  Sharded over the ranks when
        `loader` is a partitioned CSDataLoader or `distributed` is true (evaluate_main's rule); every rank gets the whole set's IU."""
        mean_IU, IU_array = evaluate_main(model=model, loader=loader, gpu_id=gpu_id, input_size=input_size, num_classes=num_classes, whole=whole,
                                          distributed=distributed)
        return mean_IU, IU_array

    def save_ckpt(self, epoch, step, mean_IU, IU_array):
        """The trained network's state_dict to <snapshot_dir>/CS_scenes_<step>_<mean_IU>.pth -> that path.  Replicas are identical:
        rank 0 writes, other ranks return None."""
        if self.world > 1 and dist.get_rank() != 0:
            return
        path = osp.join(self.args.snapshot_dir, 'CS_scenes_' + str(step) + '_' + str(mean_IU) + '.pth')
        torch.save(self._net.state_dict(), path)
        return path

    # ---- resuming a run --------------------------------------------------------------------------------------------------------
    def _trained(self):
        """[(field prefix, module, FlatSGD)]: the trained network, and NetModel's discriminator."""
        parts = [("", self._net, self.G_solver)]
        if getattr(self, "D_solver", None) is not None:
            parts.append(("D_", self.D_model, self.D_solver))
        return parts

    def _extra_states(self):
        """{field: module} saved and restored beside the trained network (NetModel: `mimic_state_dict` / `cwd_state_dict`, the MIMIC
        and CWD adapters)."""
        return {}

    def save_training_state(self, path, step, epoch=0, best_mean_IU=None, IU_array=None, loader=None):
        """Writes everything needed to continue this run after step `step` (best_mean_IU defaults to self.best_mean_IU) to `path`,
        one torch.save dict:
          * `state_dict`, `step`, `epoch`, `best_mean_IU`, `IU_array` -- the reference's checkpoint keys: renamed to model_best.pth.tar
            in S_ckpt_path / ckpt_path, the file loads through load_S_model / load_seg_model (S_resume / resume) like the reference's;
          * `D_state_dict` (spectral-norm u / v, BN buffers included), `G_solver` / `D_solver` (momentum, steps, lr, flat length);
          * with MIMIC, `mimic_state_dict`: the adapters (their momentum is in G_solver);
          * with CWD feature levels, `cwd_state_dict`: their adapters (likewise);
          * `ranks`: per rank, the torch CPU and CUDA generators, Python `random`, numpy's global generator and `loader.state_dict()`;
          * `format`, `version`, `world_size`, `kind`, `classes_num`: what load_training_state checks.
        Collective: every rank calls it.  Rank 0 writes a temporary file beside `path` and renames it over `path`, so an interrupted
        write leaves the previous file as it was; no rank returns before the file is complete (or before every rank raised)."""
        rank = dist.get_rank() if self.world > 1 else 0
        solvers = {prefix + "solver": dict(s.state_dict(), numel=s.flat_m.numel()) for prefix, _, s in self._trained()}  # collective (NVLS)
        mine = _rng_states(self.device, loader)
        ranks = [None] * self.world
        if self.world > 1:
            dist.all_gather_object(ranks, mine)
        else:
            ranks[0] = mine
        err = None
        if rank == 0:
            state = dict(format=TRAINING_STATE_FORMAT, version=TRAINING_STATE_VERSION, world_size=self.world,
                         kind=(self.kind_option, self.kind), classes_num=int(self.args.classes_num),
                         step=int(step), epoch=int(epoch), best_mean_IU=float(self.best_mean_IU if best_mean_IU is None else best_mean_IU),
                         IU_array=None if IU_array is None else np.asarray(IU_array, dtype=np.float64), ranks=ranks)
            for prefix, module, _ in self._trained():
                state[prefix + "state_dict"] = _cpu_state(module)
            for field, module in self._extra_states().items():
                state[field] = _cpu_state(module)
            state["G_solver"] = solvers["solver"]
            state["D_solver"] = solvers.get("D_solver")
            for k in ("G_solver", "D_solver"):
                if state[k] is not None:
                    state[k]["momentum"] = state[k]["momentum"].cpu()
            err = self._write_atomically(state, path)
        if self.world > 1:
            box = [err]
            dist.broadcast_object_list(box, 0)                     # doubles as the barrier: rank 0 has renamed (or failed)
            err = box[0]
        if err is not None:
            raise RuntimeError("writing the training state to %s failed: %s" % (path, err))

    @staticmethod
    def _write_atomically(state, path):
        """torch.save to a temporary file in `path`'s directory, fsync, rename over `path` -> None, or the error's text (the temporary
        file removed, `path` untouched)."""
        d = osp.dirname(osp.abspath(path))
        fd, tmp = tempfile.mkstemp(dir=d, prefix="." + osp.basename(path) + ".", suffix=".tmp")
        try:
            with os.fdopen(fd, "wb") as f:
                torch.save(state, f)
                f.flush()
                os.fsync(f.fileno())
            os.replace(tmp, path)
        except Exception as e:                                     # noqa: BLE001
            if osp.exists(tmp):
                os.remove(tmp)
            return repr(e)
        return None

    def load_training_state(self, path, loader=None):
        """Restores what save_training_state wrote, in place: the network's and the discriminator's parameters (copied into the
        existing flat buffers), BN buffers and spectral-norm u / v, both solvers' momentum, step counts and lr, and this rank's random
        generators -- so a step already captured in a CUDA graph keeps replaying, now from the restored state -- and, when `loader`
        is given, its position (CSDataLoader.load_state_dict: the next iteration yields the rest of the interrupted one).  Sets
        args.last_step / start_epoch / best_mean_IU and self.best_mean_IU -> the saved step.
        A file that does not match this model (format version, kind, classes_num, world size, flat-buffer lengths, state-dict keys or
        shapes, a loader position when `loader` is given) raises ValueError naming the field before anything is modified."""
        ck = _torch_load(path)
        rank = dist.get_rank() if self.world > 1 else 0

        def mismatch(field, got, want):
            raise ValueError("training state %s does not match the model: %s is %r, the model's %r" % (path, field, got, want))

        if not isinstance(ck, dict) or ck.get("format") != TRAINING_STATE_FORMAT:
            mismatch("format", ck.get("format") if isinstance(ck, dict) else type(ck).__name__, TRAINING_STATE_FORMAT)
        if ck.get("version") != TRAINING_STATE_VERSION:
            mismatch("version", ck.get("version"), TRAINING_STATE_VERSION)
        if tuple(ck["kind"]) != (self.kind_option, self.kind):
            mismatch("kind", tuple(ck["kind"]), (self.kind_option, self.kind))
        if ck["classes_num"] != int(self.args.classes_num):
            mismatch("classes_num", ck["classes_num"], int(self.args.classes_num))
        if ck["world_size"] != self.world:
            mismatch("world_size", ck["world_size"], self.world)
        parts = self._trained()
        for prefix, module, solver in parts:
            field = "G_solver" if prefix == "" else "D_solver"
            got = None if ck.get(field) is None else ck[field]["numel"]
            if got != solver.flat_m.numel() or tuple(ck[field]["momentum"].shape) != (solver.flat_m.numel(),):
                mismatch(field + ".numel", got, solver.flat_m.numel())
            _check_state_dict(prefix + "state_dict", module.state_dict(), ck.get(prefix + "state_dict"))
        if len(parts) == 1 and ck.get("D_solver") is not None:
            mismatch("D_solver", "a discriminator", None)
        extra = self._extra_states()
        for field, module in extra.items():
            _check_state_dict(field, module.state_dict(), ck.get(field))
        for field in ck:
            if field.endswith("_state_dict") and field not in ("state_dict", "D_state_dict") and field not in extra:
                mismatch(field, "present", None)
        mine = ck["ranks"][rank]
        if loader is not None:
            if mine.get("loader") is None:
                mismatch("ranks[%d].loader" % rank, None, "a CSDataLoader position")
            loader.load_state_dict(mine["loader"])                  # checks its fields first; sets nothing but the pending position

        with torch.no_grad():
            for prefix, module, solver in parts:
                module.load_state_dict(ck[prefix + "state_dict"])      # copy_ into the existing tensors (flat-buffer views)
                solver.load_state_dict(ck["G_solver" if prefix == "" else "D_solver"])
            for field, module in extra.items():
                module.load_state_dict(ck[field])
        _set_rng_states(mine, self.device)
        self.args.last_step, self.args.start_epoch = ck["step"], ck["epoch"]
        self.args.best_mean_IU = self.best_mean_IU = ck["best_mean_IU"]
        return ck["step"]
