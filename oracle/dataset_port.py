"""TEST INFRASTRUCTURE -- CPU restatement (numpy) of the reference's Cityscapes training loader, `dataset/datasets.py::CSDataSet`.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import anything under oracle/.  The product path
(structure_knowledge_distillation_b200/dataset + csrc/augment.cu) never does.

What it restates, and where the arithmetic lives:
  * `CSDataSet.__getitem__`                 dataset/datasets.py:170-210  (order of operations and of the RNG draws)
  * `CSDataSet.generate_scale_label`        dataset/datasets.py:155-159  (cv2.resize INTER_LINEAR / INTER_NEAREST)
  * `CSDataSet.id2trainId`                  dataset/datasets.py:161-169  (a 256-entry look-up table)
  * cv2.resize itself is a THIRD-PARTY dependency (opencv-python, 4.13.0 in this image; the reference pins no version).  Restated
    from OpenCV's published algorithm (modules/imgproc/src/resize.cpp): uint8 INTER_LINEAR = fixed-point separable interpolation,
    coefficients round(w * 2048) as int16, horizontal pass in int32, vertical pass
    `((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2`; INTER_NEAREST = `min(floor(d * (1 / f)), size - 1)`;
    destination size `cvRound(size * f)`.
PINNED: `oracle/make_golden_dataset.py` runs the UNMODIFIED reference class (cv2 4.13.0 underneath) on synthetic PNG files in this
container and stores inputs, seeds and outputs in tests/golden/dataset.pt; tests/test_dataset_cpu.py holds this port to those
outputs bit for bit (15 scale factors, padding, crop, mirror, the validation configuration).
"""
import random

import numpy as np

IGNORE = 255

# datasets.py:143-149 -- id -> trainId; ids absent from the table (and 255) pass through
ID_TO_TRAINID = {-1: IGNORE, 0: IGNORE, 1: IGNORE, 2: IGNORE, 3: IGNORE, 4: IGNORE, 5: IGNORE, 6: IGNORE, 7: 0, 8: 1, 9: IGNORE,
                 10: IGNORE, 11: 2, 12: 3, 13: 4, 14: IGNORE, 15: IGNORE, 16: IGNORE, 17: 5, 18: IGNORE, 19: 6, 20: 7, 21: 8, 22: 9,
                 23: 10, 24: 11, 25: 12, 26: 13, 27: 14, 28: 15, 29: IGNORE, 30: IGNORE, 31: 16, 32: 17, 33: 18}


def trainid_lut():
    lut = np.arange(256, dtype=np.uint8)
    for k, v in ID_TO_TRAINID.items():
        if 0 <= k < 256:
            lut[k] = v
    return lut


def cv_round(x):
    """cvRound / saturate_cast<int>(double): round half to even."""
    return int(np.rint(x))


def _linear_table(dst, f):
    """resize.cpp (resizeGeneric setup): fx = float((d + 0.5) * scale - 0.5), scale = 1 / f in double; s = floor(fx); fx -= s."""
    scale = 1.0 / f
    d = np.arange(dst, dtype=np.float64)
    fx = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(fx).astype(np.int64)
    fx = (fx - s.astype(np.float32)).astype(np.float32)
    return s, fx


def _coef(w):
    """saturate_cast<short>(w * INTER_RESIZE_COEF_SCALE): float product, round half to even."""
    return np.rint((w * np.float32(2048)).astype(np.float32)).astype(np.int64)


def resize_linear_u8(img, f):
    """cv2.resize(img, None, fx=f, fy=f, interpolation=cv2.INTER_LINEAR) for a uint8 H x W x C image."""
    H, W, _ = img.shape
    dw, dh = cv_round(W * f), cv_round(H * f)
    sx, fx = _linear_table(dw, f)
    lo = sx < 0; fx[lo] = 0; sx[lo] = 0                       # columns left of the first source pixel: weight 1 on pixel 0
    hi = sx >= W - 1; fx[hi] = 0; sx[hi] = W - 1               # ... and right of the last one
    a0, a1 = _coef(np.float32(1) - fx), _coef(fx)
    sx1 = np.minimum(sx + 1, W - 1)
    sy, fy = _linear_table(dh, f)                              # rows: indices are clipped, the weights are NOT reset
    b0, b1 = _coef(np.float32(1) - fy), _coef(fy)
    y0, y1 = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)
    S = img.astype(np.int64)
    r0 = S[y0][:, sx] * a0[None, :, None] + S[y0][:, sx1] * a1[None, :, None]
    r1 = S[y1][:, sx] * a0[None, :, None] + S[y1][:, sx1] * a1[None, :, None]
    out = (((b0[:, None, None] * (r0 >> 4)) >> 16) + ((b1[:, None, None] * (r1 >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


def resize_nearest(lab, f):
    """cv2.resize(lab, None, fx=f, fy=f, interpolation=cv2.INTER_NEAREST) for an H x W array."""
    H, W = lab.shape
    dw, dh = cv_round(W * f), cv_round(H * f)
    inv = 1.0 / f
    sx = np.minimum(np.floor(np.arange(dw) * inv).astype(np.int64), W - 1)
    sy = np.minimum(np.floor(np.arange(dh) * inv).astype(np.int64), H - 1)
    return lab[sy][:, sx]


def cs_getitem(image, label, crop_size, mean, scale=True, mirror=True, ignore_label=IGNORE, py_random=random, np_random=np.random):
    """`CSDataSet.__getitem__` after the two `cv2.imread` calls (datasets.py:173-210).

    image: H x W x 3 uint8 (BGR as cv2 reads it); label: H x W uint8 raw ids.  Draws from `py_random` and `np_random` in the
    reference's order: randint(0, 14) [scale], randint h_off, randint w_off, choice(2) [mirror].
    Returns (image float32 3 x ch x cw, label float32 ch x cw, params dict)."""
    crop_h, crop_w = crop_size
    label = trainid_lut()[label]                                                      # :175
    params = {"f_scale": 1.0, "scale_idx": -1}
    if scale:                                                                          # :178-179 -> :155-159
        k = py_random.randint(0, 14)
        f_scale = 0.7 + k / 10.0
        image, label = resize_linear_u8(image, f_scale), resize_nearest(label, f_scale)
        params.update(f_scale=f_scale, scale_idx=k)
    image = np.asarray(image, np.float32)                                              # :180
    image = image - np.asarray(mean, np.float32)                                       # :181 (float32 - float32)
    img_h, img_w = label.shape
    pad_h, pad_w = max(crop_h - img_h, 0), max(crop_w - img_w, 0)                      # :183-184
    if pad_h > 0 or pad_w > 0:                                                         # :185-191 zeros / ignore label, bottom and right
        image = np.pad(image, ((0, pad_h), (0, pad_w), (0, 0)), constant_values=0.0)
        label = np.pad(label, ((0, pad_h), (0, pad_w)), constant_values=ignore_label)
    img_h, img_w = label.shape
    h_off = py_random.randint(0, img_h - crop_h)                                       # :196-197
    w_off = py_random.randint(0, img_w - crop_w)
    image = np.asarray(image[h_off:h_off + crop_h, w_off:w_off + crop_w], np.float32)  # :199-200
    label = np.asarray(label[h_off:h_off + crop_h, w_off:w_off + crop_w], np.float32)
    image = image.transpose((2, 0, 1))                                                 # :202
    flip = 1
    if mirror:                                                                         # :203-206
        flip = int(np_random.choice(2)) * 2 - 1
        image = image[:, :, ::flip]
        label = label[:, ::flip]
    params.update(h_off=h_off, w_off=w_off, flip=flip)
    return image.copy(), label.copy(), params
