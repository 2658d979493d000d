"""`evaluate_main` of the reference (networks/evaluate.py:115-206) on the frozen-path kernels: eval-mode BN folded into the
wgmma convolution epilogues, class scores up-sampled / accumulated / arg-maxed and the confusion matrix counted on the GPU
(csrc/eval.cu); only the num_classes x num_classes counts come back to the host.

Kept: whole-image prediction at 1024x2048 (`whole=True`, predict_multiscale), with or without extra scales and the mirrored pass,
sliding 1/3-overlap tiles of `input_size` (`whole=False`, predict_sliding, single scale only), valid-region cropping by `size`,
ignore label 255, mean IU = tp / max(1, pos + res - tp), and the palette PNGs of :187-191 (`png_dir`; Cityscapes label ids for
type='test', the files the Cityscapes server scores).  `save_dir` additionally writes the cropped uint8 prediction maps as .pt."""
import os
import queue
import threading
from math import ceil

import numpy as np
import torch
import torch.distributed as dist

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


def zoom_shape(H, W, scale):
    """scipy.ndimage.zoom's output size for zoom (1, 1, s, s): round(H * s), round(W * s) with Python rounding."""
    return int(round(H * float(scale))), int(round(W * float(scale)))


def _check_scales(scales):
    scales = tuple(float(s) for s in scales)
    if not scales or any(not s > 0 for s in scales):
        raise ValueError("scales must be a non-empty sequence of positive numbers, got %r" % (scales,))
    return scales


def zoom_image(image, scale, flip=False):
    """scipy.ndimage.zoom(image, (1, 1, s, s), order=1, prefilter=False) of a float32 (1, 3, H, W) device image, bit for bit
    (evaluate.py:127), as the (1 + flip, 4, h, w) NHWC tensor Res_pspnet.forward takes; item 1 is the mirror image (:130)."""
    if image.dim() != 4 or image.shape[0] != 1 or image.shape[1] != 3:
        raise ValueError("zoom_image takes one (1, 3, H, W) image, got %s" % (tuple(image.shape),))
    image = image.float().contiguous()
    _, _, H, W = image.shape
    oh, ow = zoom_shape(H, W, scale)
    if oh < 1 or ow < 1:
        raise ValueError("scale %r leaves no pixel of a %dx%d image" % (scale, H, W))
    out = torch.empty((2 if flip else 1, oh, ow, 4), device=image.device, dtype=torch.float32)
    lib().skd_eval_zoom_image(H, W, image.data_ptr(), oh, ow, 1 if flip else 0, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return out.permute(0, 3, 1, 2)


def predict_multiscale(model, image, tile_size, scales, flip, full):
    """evaluate.py:115-134: full += the class scores up-sampled to `tile_size`, averaged over the zoomed copies of the image; with
    `flip`, each scale runs the image and its mirror as one batch-2 forward (eval-mode BN keeps the two independent) and adds
    0.5 * (scores + mirrored scores of the mirror)."""
    scales = _check_scales(scales)
    hh, ww = min(tile_size[0], full.shape[0]), min(tile_size[1], full.shape[1])
    weight = 1.0 / len(scales)
    for s in scales:
        logits = _scores(model, zoom_image(image, s, flip))
        _, c, h, w = logits.shape
        sn, sc, sp = ops.pixel_strides(logits)
        lib().skd_eval_upsample_accumulate_ms(c, h, w, logits.data_ptr(), sn, sc, sp, tile_size[0], tile_size[1], hh, ww, full.data_ptr(),
                                              full.shape[1], weight, 1 if flip else 0, torch.cuda.current_stream().cuda_stream)


def get_palette(num_cls):
    """The colour map of the prediction PNGs (evaluate.py:40-61): class j's bits, three at a time, go to the R, G and B bytes from
    the top bit down.  -> flat [r0, g0, b0, r1, ...] list of 3 * num_cls ints."""
    palette = []
    for j in range(num_cls):
        rgb, lab, bit = [0, 0, 0], j, 7
        while lab:
            for k in range(3):
                rgb[k] |= ((lab >> k) & 1) << bit
            bit -= 1
            lab >>= 3
        palette += rgb
    return palette


class _PngWriter:
    """Encodes prediction maps as palette PNGs on ONE background thread, so the host encode of image i overlaps the forward pass of
    image i + 1.  The device -> pinned host copy is queued on the current stream and the thread waits for its event.  An encode
    error is raised in the caller at the next submit() or at close()."""

    def __init__(self, palette):
        self._palette = palette
        self._q = queue.Queue(maxsize=4)
        self._error = None
        self._thread = threading.Thread(target=self._run, name="skd-png-writer", daemon=True)
        self._thread.start()

    def _run(self):
        from PIL import Image
        while True:
            item = self._q.get()
            if item is None:
                return
            if self._error is not None:
                continue
            host, done, path = item
            try:
                done.synchronize()
                im = Image.fromarray(host.numpy())
                im.putpalette(self._palette)
                im.save(path)
            except BaseException as e:      # handed to the caller
                self._error = e

    def _raise(self):
        if self._error is not None:
            err, self._error = self._error, None
            raise err

    def submit(self, pred, path):
        self._raise()
        host = torch.empty(pred.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(pred, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        self._q.put((host, done, path))

    def close(self):
        if self._thread.is_alive():
            self._q.put(None)
            self._thread.join()
        self._raise()


def _sum_over_ranks(counts):
    """All-reduce (sum) of an integer count tensor over the default process group: in place on the device under NCCL, through a
    host copy under a CPU backend (gloo)."""
    if "nccl" in str(dist.get_backend()) and counts.is_cuda:
        dist.all_reduce(counts)
        return counts
    host = counts.cpu()
    dist.all_reduce(host)
    return host


def evaluate_main(model, loader, gpu_id, input_size, num_classes, whole=False, recurrence=1, type='val', save_dir=None, scales=(1.0,),
                  flip=False, png_dir=None, distributed=False):
    """-> (mean_IU, IU_array) over `loader` batches (image (1,3,H,W), label (1,H,W), size, name); type='test' batches are
    (image, size, name), count nothing, and their output is the PNGs.

    scales / flip: predict_multiscale's (whole=True only; the reference's sliding path has neither).  The defaults run the single
    whole-image pass.  png_dir: write <png_dir>/<name>.png, the arg-max of the whole image as an 8-bit palette image
    (get_palette(256)), in Cityscapes label ids for type='test' (19 classes); with save_dir too, the .pt maps are the same values.

    Sharded evaluation: when `loader` is a partitioned `CSDataLoader` with world_size > 1, or with `distributed=True` (a caller's own
    sharded loader), every rank of the default process group calls this on its share of the images and the confusion counts are
    summed over the ranks (one all-reduce of num_classes^2 int64 counts: on the device under NCCL, through the host otherwise), so
    every rank returns the (mean_IU, IU_array) of the whole set, bit for bit the one-process result.  png_dir / save_dir files are
    written by the rank that scored the image."""
    scales = _check_scales(scales)
    from ..dataset.datasets import CSDataLoader
    sharded = bool(distributed) or (isinstance(loader, CSDataLoader) and (loader.world_size or 1) > 1)
    if sharded:
        if not (dist.is_available() and dist.is_initialized()):
            raise ValueError("sharded evaluation needs an initialised torch.distributed process group")
        if isinstance(loader, CSDataLoader) and loader.world_size is not None and loader.world_size != dist.get_world_size():
            raise ValueError("the loader is partitioned over %d ranks, the process group has %d" % (loader.world_size, dist.get_world_size()))
    multi = scales != (1.0,) or bool(flip)
    if multi and not whole:
        raise ValueError("scales other than (1.0,) and flip need whole=True: the sliding-window path is single-scale")
    if png_dir is not None and type == 'test' and num_classes != 19:
        raise ValueError("Cityscapes label-id PNGs need the 19 train ids, got num_classes=%d" % num_classes)
    h, w = map(int, input_size.split(',')) if isinstance(input_size, str) else input_size
    tile = (1024, 2048) if whole else (h, w)
    dev = next(model.parameters()).device
    if dev.type != 'cuda':                                   # evaluate.py:166: the reference moves the model itself
        model.cuda()
        dev = next(model.parameters()).device
    was_training = model.training
    model.eval()
    conf = torch.zeros(num_classes, num_classes, device=dev, dtype=torch.int64)
    L = lib()
    writer = lut = None
    if png_dir is not None:
        os.makedirs(png_dir, exist_ok=True)
        if type == 'test':
            from ..dataset.datasets import cityscapes_id_tables
            lut = torch.from_numpy(cityscapes_id_tables()[1]).to(dev)
        writer = _PngWriter(get_palette(256))
    try:
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
            if whole and multi:
                predict_multiscale(model, image, tile, scales, flip, full)
            elif whole:
                predict_whole(model, image, tile, full)
            else:
                predict_sliding(model, image, tile, full)
            vh, vw = int(min(size[0], H)), int(min(size[1], W))
            gt = None
            if label is not None:
                gt = torch.as_tensor(label)[0].to(dev).long().contiguous()
            st = torch.cuda.current_stream().cuda_stream
            if writer is None:
                pred = torch.empty(H, W, device=dev, dtype=torch.uint8) if save_dir else None
                L.skd_eval_argmax_confusion(H, W, num_classes, full.data_ptr(), None if gt is None else gt.data_ptr(), 0 if gt is None else gt.shape[1], vh, vw,
                                            255, conf.data_ptr(), None if pred is None else pred.data_ptr(), st)
            else:
                pred = torch.empty(H, W, device=dev, dtype=torch.uint8)          # the whole image (:187-191), not the `size` crop
                L.skd_eval_argmax_confusion_lut(H, W, num_classes, full.data_ptr(), None if gt is None else gt.data_ptr(),
                                                0 if gt is None else gt.shape[1], vh, vw, 255, conf.data_ptr(), pred.data_ptr(), H, W,
                                                None if lut is None else lut.data_ptr(), st)
                writer.submit(pred, os.path.join(png_dir, str(name[0]) + '.png'))
            if save_dir:
                os.makedirs(save_dir, exist_ok=True)
                torch.save(pred[:vh, :vw].cpu(), os.path.join(save_dir, str(name[0]) + '.pt'))
    finally:
        if writer is not None:
            writer.close()
        if was_training:
            model.train()
    if sharded:
        conf = _sum_over_ranks(conf)
    cm = conf.cpu().numpy().astype(np.float64)
    pos, res, tp = cm.sum(1), cm.sum(0), np.diag(cm)
    IU_array = tp / np.maximum(1.0, pos + res - tp)
    return IU_array.mean(), IU_array
