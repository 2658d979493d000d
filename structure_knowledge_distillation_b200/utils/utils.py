"""Helpers with the reference's names (utils/utils.py): the affinity function of the pair-wise loss (:170-183) and the
checkpoint loaders NetModel's constructor calls (:73-151).  Checkpoints written by the reference load unchanged: parameter
names and shapes are the reference's (convolution weights are merely STORED channels-last, which a state dict does not see)."""
import logging
import os
import shutil

import torch

from .. import functions as Fn


def sim_dis_compute(f_S, f_T):
    """sum((A_T - A_S)^2) / nodes^2 / N on already-pooled features (utils/utils.py:180-183).  The affinity matrices are
    never returned to Python: pooling with a 1x1 window is the identity, the rest is the fused gram/L2 kernel."""
    return Fn.PairWiseLoss.apply(f_S, f_T.detach(), 1, 1)


def _torch_load(path):
    """torch.load restricted to tensors / plain containers; numpy arrays (the reference stores `IU_array`) are allow-listed."""
    allow = []
    try:
        import numpy as np
        core = getattr(np, "_core", None) or getattr(np, "core", None)
        allow = [np.ndarray, np.dtype, core.multiarray._reconstruct]
        allow += [type(np.dtype(t)) for t in (np.float64, np.float32, np.int64, np.int32, np.uint8, np.bool_)]
    except Exception:                                                      # noqa: BLE001
        pass
    try:
        with torch.serialization.safe_globals(allow):
            return torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:                                                 # noqa: BLE001
        raise RuntimeError("refusing to unpickle %s with weights_only=True (%s); convert the checkpoint to plain tensors" % (path, e))


def _strip_module(state_dict, with_module):
    """`with_module == False`: keys were saved from an nn.DataParallel wrapper, drop the leading 'module.' (utils.py:124-127)."""
    if with_module:
        return state_dict
    return {(k[7:] if k.startswith("module.") else k): v for k, v in state_dict.items()}


def load_T_model(model, ckpt_path):
    """utils/utils.py:73-91: remap `head.0.*` -> `pspmodule.*`, `head.1.*` -> `head.*`, drop `fc.*`."""
    if ckpt_path and os.path.exists(ckpt_path):
        saved = _torch_load(ckpt_path)
        new = model.state_dict().copy()
        for k, v in saved.items():
            if k.startswith('fc.'):
                continue
            if k.startswith('head.0.'):
                new['pspmodule.' + k[7:]] = v
            elif k.startswith('head.1.'):
                new['head.' + k[7:]] = v
            else:
                new[k] = v
        model.load_state_dict(new)
        logging.info("load" + str(ckpt_path))
        return True
    logging.info("=> no teacher ckpt find")
    return False


def _encoder_only(model, state):
    """True when `model` is the full ESPNet and `state` an ESPNet-C state dict (its keys without the `encoder.` prefix): training the
    encoder first, then the whole network, is the usual way to train ESPNet."""
    enc = getattr(model, "encoder", None)
    return enc is not None and not any(k.startswith("encoder.") for k in state) and set(state) <= set(enc.state_dict())


def load_S_model(args, model, with_module=True):
    """utils/utils.py:93-127: ImageNet initialisation (key intersection) when `is_student_load_imgnet`, else resume from
    `<S_ckpt_path>/model_best.pth.tar` when `S_resume` -- restoring last_step / start_epoch / best_mean_IU into `args`.  The full
    ESPNet student also takes an ESPNet-C state dict, loaded under `encoder.` (the decoder keeps its initialisation)."""
    ckpt_dir = getattr(args, "S_ckpt_path", "")
    if ckpt_dir and not os.path.exists(ckpt_dir):
        os.makedirs(ckpt_dir, exist_ok=True)
    if getattr(args, "is_student_load_imgnet", False):
        path = str(getattr(args, "student_pretrain_model_imgnet", ""))
        if os.path.isfile(path):
            saved = _torch_load(path)
            if _encoder_only(model, saved):
                saved = {"encoder." + k: v for k, v in saved.items()}
            new = model.state_dict()
            new.update({k: v for k, v in saved.items() if k in new})
            model.load_state_dict(new)
            logging.info("=> load" + path)
            return "imagenet"
        logging.info("=> the pretrain model on imgnet '{}' does not exit".format(path))
        return None
    if getattr(args, "S_resume", False) and ckpt_dir:
        file = ckpt_dir + '/model_best.pth.tar'
        if os.path.isfile(file):
            ck = _torch_load(file)
            args.last_step = ck.get('step')
            args.start_epoch = ck.get('epoch')
            args.best_mean_IU = ck.get('best_mean_IU')
            state = _strip_module(ck['state_dict'], with_module)
            (model.encoder if _encoder_only(model, state) else model).load_state_dict(state)
            logging.info("=> loaded checkpoint '{}' \n (epoch:{} step:{} best_mean_IU:{} \n )".format(file, args.start_epoch, args.last_step,
                                                                                              args.best_mean_IU))
            return "resume"
        logging.info("=> checkpoint '{}' does not exit".format(file))
    return None


def load_D_model(args, model, with_module=True):
    """utils/utils.py:129-151."""
    ckpt_dir = getattr(args, "D_ckpt_path", "")
    if getattr(args, "D_resume", False) and ckpt_dir:
        if not os.path.exists(ckpt_dir):
            os.makedirs(ckpt_dir, exist_ok=True)
        file = ckpt_dir + '/model_best.pth.tar'
        if os.path.isfile(file):
            ck = _torch_load(file)
            args.start_epoch = ck['epoch']
            args.best_mean_IU = ck['best_mean_IU']
            model.load_state_dict(_strip_module(ck['state_dict'], with_module))
            logging.info("=> loaded checkpoint '{}' (epoch {})".format(file, ck['epoch']))
            return "resume"
        logging.info("=> checkpoint '{}' does not exit".format(file))
    return None


def save_checkpoint(state, is_best, fdir):
    """utils/utils.py:153-157."""
    filepath = os.path.join(fdir, 'checkpoint.pth')
    torch.save(state, filepath)
    if is_best:
        shutil.copyfile(filepath, os.path.join(fdir, 'model_best.pth.tar'))
