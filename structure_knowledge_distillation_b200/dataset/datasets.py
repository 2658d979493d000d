"""Cityscapes training loader with the augmentation on the GPU -- host-side mirror of `dataset/datasets.py::CSDataSet`
(reference dataset/datasets.py:121-210) for the callers of the hot path (`train_and_eval.py:13-17` builds the loaders whose batches
go to `NetModel.set_input`).

Split of the work:
  * worker processes (`CSDataSet.__getitem__`): `cv2.imread` of the image / label files, and the RANDOM DRAWS -- scale index, crop origin,
    mirror -- from `random` / `np.random` in exactly the reference's order (datasets.py:156,196-197,204), so a seeded run sees the same
    augmentations as the reference.  Nothing is resized, converted to float, padded or copied on the CPU.
  * the GPU (`DeviceAugment` -> `skd_cs_augment_batch`, csrc/augment.cu): one kernel per batch produces the float32 CHW crop and the
    label crop directly from the raw uint8 files, bit-exact with the reference's cv2 pipeline (tests/test_dataset_gpu.py).
`CSDataLoader` chains the two and yields `(images, labels, size, name)` batches resident on the device, i.e. what `set_input` takes.
There is no CPU fallback: without libskd_b200.so `DeviceAugment` raises at import of the ops.
"""
import collections
import ctypes
import os.path as osp
import random

import numpy as np
import torch
from torch.utils import data

IGNORE_LABEL = 255

Augmentation = collections.namedtuple("Augmentation", "scale_idx f_scale scaled_h scaled_w h_off w_off flip")


def _cv_round(x):
    """cvRound (round half to even): cv2.resize's destination size for a scale factor."""
    return int(np.rint(x))


def draw_augmentation(src_h, src_w, crop_size, scale=True, mirror=True):
    """The random numbers of one `CSDataSet.__getitem__` call, drawn in the reference's order from the same generators:
    `random.randint(0, 14)` (datasets.py:156), `random.randint` for h_off then w_off (:196-197), `np.random.choice(2)` (:204)."""
    crop_h, crop_w = crop_size
    scale_idx, f_scale, sh, sw = -1, 1.0, src_h, src_w
    if scale:
        scale_idx = random.randint(0, 14)
        f_scale = 0.7 + scale_idx / 10.0
        sh, sw = _cv_round(src_h * f_scale), _cv_round(src_w * f_scale)
    img_h, img_w = max(sh, crop_h), max(sw, crop_w)                    # after padding (:183-193)
    h_off = random.randint(0, img_h - crop_h)
    w_off = random.randint(0, img_w - crop_w)
    flip = 1
    if mirror:
        flip = int(np.random.choice(2)) * 2 - 1
    return Augmentation(scale_idx, f_scale, sh, sw, h_off, w_off, flip)


class CSDataSet(data.Dataset):
    """Same constructor as the reference (datasets.py:122).  `__getitem__` returns the RAW decoded files and the drawn augmentation:
    (image uint8 H x W x 3 BGR, label uint8 H x W, aug float64[7], size int[3], name)."""

    def __init__(self, root, list_path, max_iters=None, crop_size=(321, 321), mean=(128, 128, 128), scale=True, mirror=True, ignore_label=255):
        self.root, self.list_path = root, list_path
        self.crop_h, self.crop_w = crop_size
        self.scale, self.is_mirror, self.ignore_label = scale, mirror, ignore_label
        self.mean = mean
        self.img_ids = [i_id.strip().split() for i_id in open(list_path)]
        if max_iters is not None:
            self.img_ids = self.img_ids * int(np.ceil(float(max_iters) / len(self.img_ids)))
        self.files = []
        for image_path, label_path in self.img_ids:
            self.files.append({"img": osp.join(self.root, image_path), "label": osp.join(self.root, label_path),
                               "name": osp.splitext(osp.basename(label_path))[0]})
        print('{} images are loaded!'.format(len(self.img_ids)))

    def __len__(self):
        return len(self.files)

    def __getitem__(self, index):
        import cv2                                                      # decode stays on the host, as in the reference (:172-173)
        f = self.files[index]
        image = cv2.imread(f["img"], cv2.IMREAD_COLOR)
        label = cv2.imread(f["label"], cv2.IMREAD_GRAYSCALE)
        if image is None or label is None:
            raise IOError("cannot read %s / %s" % (f["img"], f["label"]))
        aug = draw_augmentation(image.shape[0], image.shape[1], (self.crop_h, self.crop_w), self.scale, self.is_mirror)
        return (torch.from_numpy(image), torch.from_numpy(label), torch.tensor(aug, dtype=torch.float64), np.array(image.shape), f["name"])


class _Sample(ctypes.Structure):          # include/skd.h: skd_cs_sample
    _fields_ = [("image", ctypes.c_void_p), ("label", ctypes.c_void_p), ("src_h", ctypes.c_int), ("src_w", ctypes.c_int),
                ("f_scale", ctypes.c_double), ("scaled_h", ctypes.c_int), ("scaled_w", ctypes.c_int), ("h_off", ctypes.c_int),
                ("w_off", ctypes.c_int), ("flip", ctypes.c_int)]


class DeviceAugment:
    """raw batch -> (images float32 [B,3,crop_h,crop_w], labels [B,crop_h,crop_w]) on the device, one kernel launch.

    `label_dtype`: torch.float32 is what the reference's `__getitem__` returns; torch.int64 is what `NetModel.set_input` makes of it
    (`labels.long()`, kd_model.py:105) -- the default, it saves that conversion pass."""

    def __init__(self, crop_size, mean, ignore_label=IGNORE_LABEL, label_dtype=torch.int64, device=None):
        from .. import _cabi
        self._lib = _cabi.lib()
        self.crop_h, self.crop_w = crop_size
        self.mean = (ctypes.c_float * 3)(*[float(np.float32(m)) for m in mean])
        self.ignore_label = int(ignore_label)
        assert label_dtype in (torch.int64, torch.float32)
        self.label_dtype = label_dtype
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self._keep = None

    def _to_device_list(self, x):
        if torch.is_tensor(x):                                               # a stacked batch travels in one copy
            d = x.to(self.device, non_blocking=True).contiguous()
            return [d[i] for i in range(d.shape[0])]
        return [t.to(self.device, non_blocking=True).contiguous() for t in x]

    def __call__(self, images, labels, augs):
        """images: uint8 [B,H,W,3] tensor or list of [H,W,3]; labels: uint8 [B,H,W] or list; augs: [B,7] rows of `Augmentation`."""
        dev_i, dev_l = self._to_device_list(images), self._to_device_list(labels)
        n = len(dev_i)
        arr = (_Sample * n)()
        for i in range(n):
            if dev_i[i].dtype != torch.uint8 or dev_l[i].dtype != torch.uint8 or dev_i[i].dim() != 3 or dev_i[i].shape[2] != 3:
                raise ValueError("raw image must be uint8 H x W x 3 and raw label uint8 H x W")
            a = [float(v) for v in augs[i]]
            s = arr[i]
            s.image, s.label = dev_i[i].data_ptr(), dev_l[i].data_ptr()
            s.src_h, s.src_w = int(dev_i[i].shape[0]), int(dev_i[i].shape[1])
            s.f_scale = a[1] if a[0] >= 0 else 0.0
            s.scaled_h, s.scaled_w, s.h_off, s.w_off, s.flip = int(a[2]), int(a[3]), int(a[4]), int(a[5]), int(a[6])
        out_i = torch.empty((n, 3, self.crop_h, self.crop_w), dtype=torch.float32, device=self.device)
        out_l = torch.empty((n, self.crop_h, self.crop_w), dtype=self.label_dtype, device=self.device)
        self._lib.skd_cs_augment_batch(n, ctypes.cast(arr, ctypes.c_void_p), self.crop_h, self.crop_w, ctypes.cast(self.mean, ctypes.c_void_p),
                                       self.ignore_label, out_i.data_ptr(), out_l.data_ptr(), 1 if self.label_dtype == torch.int64 else 0,
                                       torch.cuda.current_stream().cuda_stream)
        self._keep = (dev_i, dev_l)                                          # raw buffers stay referenced until the next batch
        return out_i, out_l


def _collate(batch):
    """default collate, except that raw files of different sizes stay lists"""
    imgs, labs, augs, sizes, names = zip(*batch)
    same = all(i.shape == imgs[0].shape for i in imgs)
    return (torch.stack(imgs) if same else list(imgs), torch.stack(labs) if same else list(labs), torch.stack(augs),
            torch.from_numpy(np.stack(sizes)), list(names))


class CSDataLoader:
    """Drop-in for `data.DataLoader(CSDataSet(...), batch_size=..., shuffle=True, num_workers=4, pin_memory=True)` of
    train_and_eval.py:13-15: iterating it yields `(images, labels, size, name)` with images / labels already augmented and on the GPU."""

    def __init__(self, dataset, batch_size=1, shuffle=False, num_workers=0, pin_memory=True, drop_last=False, label_dtype=torch.int64,
                 device=None):
        self.dataset = dataset
        self.loader = data.DataLoader(dataset, batch_size=batch_size, shuffle=shuffle, num_workers=num_workers, pin_memory=pin_memory,
                                      drop_last=drop_last, collate_fn=_collate)
        self.augment = DeviceAugment((dataset.crop_h, dataset.crop_w), dataset.mean, dataset.ignore_label, label_dtype, device)

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for images, labels, augs, sizes, names in self.loader:
            out_i, out_l = self.augment(images, labels, augs)
            yield out_i, out_l, sizes, names
