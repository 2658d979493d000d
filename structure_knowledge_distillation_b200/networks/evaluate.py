"""`evaluate_main` of the reference (networks/evaluate.py:162-206) on the frozen-path kernels: eval-mode BN folded into the
wgmma convolution epilogues, class scores up-sampled / accumulated / arg-maxed and the confusion matrix counted on the GPU
(csrc/eval.cu); only the num_classes x num_classes counts come back to the host.

Kept: whole-image prediction at 1024x2048 (`whole=True`, predict_multiscale with scale 1.0, no flip) and sliding 1/3-overlap
tiles of `input_size` (`whole=False`, predict_sliding), valid-region cropping by `size`, ignore label 255, mean IU =
tp / max(1, pos + res - tp).  Not kept: writing colour PNGs to ./outputs (pass `save_dir` to get uint8 label maps as .pt)."""
import os
from math import ceil

import numpy as np
import torch

from .. import ops
from .._cabi import lib


def _scores(model, image):
    with torch.no_grad():
        out = model(image)
    return out[0] if isinstance(out, (list, tuple)) else out


def _accumulate(full, logits, tile_hw, valid_hw, y1, x1):
    _, c, h, w = logits.shape
    sn, sc, sp = ops.pixel_strides(logits)
    lib().skd_eval_upsample_accumulate(c, h, w, logits.data_ptr(), sc, sp, tile_hw[0], tile_hw[1], valid_hw[0], valid_hw[1], full.data_ptr(),
                                       full.shape[1], y1, x1, torch.cuda.current_stream().cuda_stream)


def predict_whole(model, image, tile_size, full):
    """evaluate.py:115-122: one forward of the whole image, scores up-sampled to `tile_size`."""
    logits = _scores(model, image)
    hh, ww = min(tile_size[0], full.shape[0]), min(tile_size[1], full.shape[1])
    _accumulate(full, logits, tile_size, (hh, ww), 0, 0)


def predict_sliding(model, image, tile_size, full):
    """evaluate.py:86-113: tiles of `tile_size` with 1/3 overlap; overlapping scores are summed (arg-max is invariant to the count)."""
    _, _, H, W = image.shape
    stride = ceil(tile_size[0] * (1 - 1 / 3))
    rows = int(ceil((H - tile_size[0]) / stride) + 1)
    cols = int(ceil((W - tile_size[1]) / stride) + 1)
    for r in range(rows):
        for c in range(cols):
            x1, y1 = int(c * stride), int(r * stride)
            x2, y2 = min(x1 + tile_size[1], W), min(y1 + tile_size[0], H)
            x1, y1 = max(int(x2 - tile_size[1]), 0), max(int(y2 - tile_size[0]), 0)
            img = image[:, :, y1:y2, x1:x2]
            if img.shape[2] != tile_size[0] or img.shape[3] != tile_size[1]:                  # pad_image (evaluate.py:68-73)
                pad = torch.zeros(1, img.shape[1], tile_size[0], tile_size[1], device=img.device, dtype=img.dtype)
                pad[:, :, :img.shape[2], :img.shape[3]] = img
                img_in = pad
            else:
                img_in = img
            logits = _scores(model, img_in.contiguous())
            _accumulate(full, logits, tile_size, (img.shape[2], img.shape[3]), y1, x1)


def evaluate_main(model, loader, gpu_id, input_size, num_classes, whole=False, recurrence=1, type='val', save_dir=None):
    """-> (mean_IU, IU_array) over `loader` batches (image (1,3,H,W), label (1,H,W), size, name)."""
    h, w = map(int, input_size.split(',')) if isinstance(input_size, str) else input_size
    tile = (1024, 2048) if whole else (h, w)
    dev = next(model.parameters()).device
    was_training = model.training
    model.eval()
    conf = torch.zeros(num_classes, num_classes, device=dev, dtype=torch.int64)
    L = lib()
    for batch in loader:
        if type == 'val':
            image, label, size, name = batch
        else:
            image, size, name = batch
            label = None
        size = np.asarray(size[0])
        image = torch.as_tensor(image).float().to(dev)
        H, W = image.shape[2], image.shape[3]
        full = torch.zeros(H, W, num_classes, device=dev, dtype=torch.float32)
        if whole:
            predict_whole(model, image, tile, full)
        else:
            predict_sliding(model, image, tile, full)
        vh, vw = int(min(size[0], H)), int(min(size[1], W))
        gt = None
        if label is not None:
            gt = torch.as_tensor(label)[0].to(dev).long().contiguous()
        pred = torch.empty(H, W, device=dev, dtype=torch.uint8) if save_dir else None
        L.skd_eval_argmax_confusion(H, W, num_classes, full.data_ptr(), None if gt is None else gt.data_ptr(), 0 if gt is None else gt.shape[1], vh, vw,
                                    255, conf.data_ptr(), None if pred is None else pred.data_ptr(), torch.cuda.current_stream().cuda_stream)
        if save_dir:
            os.makedirs(save_dir, exist_ok=True)
            torch.save(pred[:vh, :vw].cpu(), os.path.join(save_dir, str(name[0]) + '.pt'))
    if was_training:
        model.train()
    cm = conf.cpu().numpy().astype(np.float64)
    pos, res, tp = cm.sum(1), cm.sum(0), np.diag(cm)
    IU_array = tp / np.maximum(1.0, pos + res - tp)
    return IU_array.mean(), IU_array
