"""TEST INFRASTRUCTURE -- CPU restatement (numpy) of the reference's PASCAL VOC loaders, `dataset/datasets.py::VOCDataSet` and
`VOCDataTestSet`, on top of oracle/dataset_port.py's cv2.resize restatement.

Only tests/ may import anything under oracle/.  The product path (structure_knowledge_distillation_b200/dataset +
csrc/augment.cu) never does.

What it restates:
  * `VOCDataSet.__getitem__`                dataset/datasets.py:45-81  (order of operations and of the RNG draws; no label table)
  * `VOCDataSet.generate_scale_label`       dataset/datasets.py:39-43  (f_scale = 0.5 + randint(0, 11) / 10.0)
  * `VOCDataTestSet.__getitem__`            dataset/datasets.py:103-119 (mean subtraction, zero padding, no crop)
The mean is subtracted by numpy itself, `float32 image -= mean`, so its type decides the arithmetic exactly as in the reference:
float32 for a float32 array, double (rounded once) for a tuple of Python numbers.
PINNED: `oracle/make_golden_voc.py` runs the UNMODIFIED reference classes on synthetic JPEG / PNG files and stores inputs, seeds
and outputs in tests/golden/voc_dataset.pt.gz; tests/test_voc_cpu.py holds this port to those outputs bit for bit.
"""
import random

import numpy as np

from .dataset_port import IGNORE, resize_linear_u8, resize_nearest


def voc_f_scale(k):
    return 0.5 + k / 10.0                                                               # datasets.py:40


def voc_getitem(image, label, crop_size, mean, scale=True, mirror=True, ignore_label=IGNORE, py_random=random, np_random=np.random):
    """`VOCDataSet.__getitem__` after the two `cv2.imread` calls.  image: H x W x 3 uint8 BGR; label: H x W uint8 class ids.
    Draws randint(0, 11) [scale], randint h_off, randint w_off, choice(2) [mirror].
    Returns (image float32 3 x ch x cw, label float32 ch x cw, params dict)."""
    crop_h, crop_w = crop_size
    params = {"f_scale": 1.0, "scale_idx": -1}
    if scale:                                                                           # :51-52 -> :39-43
        k = py_random.randint(0, 11)
        f_scale = voc_f_scale(k)
        image, label = resize_linear_u8(image, f_scale), resize_nearest(label, f_scale)
        params.update(f_scale=f_scale, scale_idx=k)
    image = np.asarray(image, np.float32)                                               # :53
    image -= mean                                                                       # :54 (numpy's promotion of `mean`)
    img_h, img_w = label.shape
    pad_h, pad_w = max(crop_h - img_h, 0), max(crop_w - img_w, 0)                       # :56-66
    if pad_h > 0 or pad_w > 0:
        image = np.pad(image, ((0, pad_h), (0, pad_w), (0, 0)), constant_values=0.0)
        label = np.pad(label, ((0, pad_h), (0, pad_w)), constant_values=ignore_label)
    img_h, img_w = label.shape
    h_off = py_random.randint(0, img_h - crop_h)                                        # :69-70
    w_off = py_random.randint(0, img_w - crop_w)
    image = np.asarray(image[h_off:h_off + crop_h, w_off:w_off + crop_w], np.float32)   # :72-73
    label = np.asarray(label[h_off:h_off + crop_h, w_off:w_off + crop_w], np.float32)
    image = image.transpose((2, 0, 1))                                                  # :75
    flip = 1
    if mirror:                                                                          # :76-79
        flip = int(np_random.choice(2)) * 2 - 1
        image = image[:, :, ::flip]
        label = label[:, ::flip]
    params.update(h_off=h_off, w_off=w_off, flip=flip)
    return image.copy(), label.copy(), params


def voc_test_getitem(image, crop_size, mean):
    """`VOCDataTestSet.__getitem__` after `cv2.imread`: -> float32 3 x max(H, crop_h) x max(W, crop_w)."""
    crop_h, crop_w = crop_size
    image = np.asarray(image, np.float32)                                               # :108-109
    image -= mean
    img_h, img_w, _ = image.shape
    pad_h, pad_w = max(crop_h - img_h, 0), max(crop_w - img_w, 0)                       # :111-117
    if pad_h > 0 or pad_w > 0:
        image = np.pad(image, ((0, pad_h), (0, pad_w), (0, 0)), constant_values=0.0)
    return image.transpose((2, 0, 1))                                                   # :118
