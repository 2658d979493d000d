"""Cityscapes and PASCAL VOC training loaders with the augmentation on the GPU -- host-side mirrors of `dataset/datasets.py::CSDataSet`
(reference dataset/datasets.py:121-210) and `VOCDataSet` (:12-81) for the callers of the hot path (`train_and_eval.py:13-17` builds the loaders whose batches
go to `NetModel.set_input`).

Split of the work:
  * worker processes (`CSDataSet.__getitem__`): `cv2.imread` of the image / label files, and the RANDOM DRAWS -- scale index, crop origin,
    mirror -- from `random` / `np.random` in exactly the reference's order (datasets.py:156,196-197,204), so a seeded run sees the same
    augmentations as the reference.  Nothing is resized, converted to float, padded or copied on the CPU.
  * the GPU (`DeviceAugment` -> `skd_augment_batch`, csrc/augment.cu): one kernel per batch produces the float32 CHW crop and the
    label crop directly from the raw uint8 files, bit-exact with the reference's cv2 pipeline (tests/test_dataset_gpu.py).
`CSDataLoader` chains the two and yields `(images, labels, size, name)` batches resident on the device, i.e. what `set_input` takes.
`VOCDataSet` differs only in its file layout, its scale rule (`VOC_SCALES`), no label table (class ids 0..20 and 255 pass through)
and its mean, which is subtracted with numpy's type as the reference does (`numpy_mean`); the same kernel serves both.
`CamVidDataSet` is `CSDataSet` with the SegNet CamVid label table (11 classes); `class_frequency_weights` gives ENet class weights
for the task loss of any of these datasets.
The test split (`CSDataTestSet`, reference datasets.py:212-250) works the same way: raw files from the workers, mean subtraction and
padding on the GPU (`DeviceTestPreprocess` -> `skd_cs_test_preprocess`), and `CSDataLoader` yields `(images, size, name)`, the
batches `evaluate_main(type='test')` unpacks.  `VOCDataTestSet` (:84-119) subtracts its own mean and yields `(images, name, size)`.
There is no CPU fallback: without libskd_b200.so `DeviceAugment` raises at import of the ops.
"""
import collections
import ctypes
import os.path as osp
import random
import struct

import numpy as np
import torch
from torch.utils import data

IGNORE_LABEL = 255

Augmentation = collections.namedtuple("Augmentation", "scale_idx f_scale scaled_h scaled_w h_off w_off flip")


def _cv_round(x):
    """cvRound (round half to even): cv2.resize's destination size for a scale factor."""
    return int(np.rint(x))


# scale rules (first factor, largest index): f_scale = first + randint(0, largest) / 10.0
CS_SCALES = (0.7, 14)                     # CSDataSet.generate_scale_label (datasets.py:158)
VOC_SCALES = (0.5, 11)                    # VOCDataSet.generate_scale_label (datasets.py:40)


def draw_augmentation(src_h, src_w, crop_size, scale=True, mirror=True, scales=CS_SCALES, py_random=random, np_random=np.random):
    """The random numbers of one `CSDataSet.__getitem__` call (`VOCDataSet` with scales=VOC_SCALES), drawn in the reference's order
    from the same generators: `random.randint(0, 14)` (datasets.py:156; VOC: randint(0, 11), :40), `random.randint` for h_off then
    w_off (:196-197), `np.random.choice(2)` (:204).  `py_random` / `np_random` replace the module-level `random` / `np.random`
    streams (a `random.Random` and a `np.random.RandomState`, as `keyed_generators` returns)."""
    crop_h, crop_w = crop_size
    scale_idx, f_scale, sh, sw = -1, 1.0, src_h, src_w
    if scale:
        scale_idx = py_random.randint(0, scales[1])
        f_scale = scales[0] + scale_idx / 10.0
        sh, sw = _cv_round(src_h * f_scale), _cv_round(src_w * f_scale)
    img_h, img_w = max(sh, crop_h), max(sw, crop_w)                    # after padding (:183-193)
    h_off = py_random.randint(0, img_h - crop_h)
    w_off = py_random.randint(0, img_w - crop_w)
    flip = 1
    if mirror:
        flip = int(np_random.choice(2)) * 2 - 1
    return Augmentation(scale_idx, f_scale, sh, sw, h_off, w_off, flip)


# The first spawn-key word keeps the permutation's stream and the draws' streams apart; numpy pads the seed's words before the key,
# so no two (seed, key) pairs share a stream.
_ORDER_KEY, _DRAW_KEY = 0, 1


def partition_order(n, seed, iteration, shuffle=True):
    """-> the sample order of iteration `iteration` of a partitioned `CSDataLoader` over `n` samples: a permutation of range(n)
    keyed by (seed, iteration), or the identity without `shuffle`.  The same on every rank and in every process."""
    if not shuffle:
        return list(range(n))
    ss = np.random.SeedSequence(seed, spawn_key=(_ORDER_KEY, iteration, 0))
    return np.random.Generator(np.random.PCG64(ss)).permutation(n).tolist()


def keyed_generators(seed, iteration, position):
    """-> (random.Random, np.random.RandomState) for the augmentation draws of the sample at global position `position` of
    iteration `iteration` of a partitioned `CSDataLoader` seeded with `seed`: fixed by the key alone, whichever rank or worker
    loads the sample."""
    words = np.random.SeedSequence(seed, spawn_key=(_DRAW_KEY, iteration, position)).generate_state(8)
    return random.Random(int.from_bytes(words[:4].astype("<u4").tobytes(), "little")), np.random.RandomState(words[4:])


_SOF = {0xC0, 0xC1, 0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF}


def _header_size(path):
    """(height, width) of a PNG or JPEG file from its header, or None when the header does not settle what `cv2.imread(path,
    IMREAD_COLOR)` returns: another format, or EXIF data, whose orientation tag cv2 applies (it may swap the two)."""
    with open(path, "rb") as f:
        head = f.read(8)
        if head == b"\x89PNG\r\n\x1a\n":
            size = None
            while True:
                chunk = f.read(8)
                if len(chunk) < 8:
                    return None
                n, typ = struct.unpack(">I4s", chunk)
                if typ == b"IHDR":
                    w, h = struct.unpack(">II", f.read(8))
                    size = (h, w)
                    f.seek(n - 8 + 4, 1)
                elif typ == b"eXIf":
                    return None
                elif typ == b"IDAT":
                    return size
                else:
                    f.seek(n + 4, 1)
        if head[:2] != b"\xff\xd8":
            return None
        f.seek(2)
        while True:
            b = f.read(1)
            while b == b"\xff":                                          # fill bytes before a marker
                m = f.read(1)
                if m != b"\xff":
                    break
            else:
                return None
            if not m:
                return None
            m = m[0]
            if m == 0x01 or 0xD0 <= m <= 0xD8:                          # markers without a length
                continue
            if m == 0xD9:                                                # end of image before any frame header
                return None
            seg = f.read(2)
            if len(seg) < 2:
                return None
            n = struct.unpack(">H", seg)[0]
            if m in _SOF:
                _, h, w = struct.unpack(">BHH", f.read(5))
                return h, w
            if m == 0xE1 and f.read(6) == b"Exif\x00\x00":
                return None
            if m == 0xE1:
                f.seek(n - 2 - 6, 1)
            else:
                f.seek(n - 2, 1)


def image_size(path):
    """(height, width) of the image `cv2.imread(path, cv2.IMREAD_COLOR)` returns.  Read from the PNG / JPEG header (no decode); other
    formats and files with EXIF data are decoded in full (for a 2048 x 1024 PNG, the cost of one `__getitem__`'s image read)."""
    size = _header_size(path)
    if size is not None:
        return size
    import cv2
    image = cv2.imread(path, cv2.IMREAD_COLOR)
    if image is None:
        raise IOError("cannot read %s" % path)
    return image.shape[:2]


class CSDataSet(data.Dataset):
    """Same constructor as the reference (datasets.py:122).  `__getitem__` returns the RAW decoded files and the drawn augmentation:
    (image uint8 H x W x 3 BGR, label uint8 H x W, aug float64[7], size int[3], name)."""

    scales = CS_SCALES

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
        return _training_sample(self, index)


def _training_sample(ds, index, py_random=random, np_random=np.random):
    """`__getitem__` of a training set (CSDataSet, CamVidDataSet, VOCDataSet) with its draws from the given streams."""
    import cv2                                                          # decode stays on the host, as in the reference (:172-173)
    f = ds.files[index]
    image = cv2.imread(f["img"], cv2.IMREAD_COLOR)
    label = cv2.imread(f["label"], cv2.IMREAD_GRAYSCALE)
    if image is None or label is None:
        raise IOError("cannot read %s / %s" % (f["img"], f["label"]))
    aug = draw_augmentation(image.shape[0], image.shape[1], (ds.crop_h, ds.crop_w), ds.scale, ds.is_mirror, ds.scales, py_random, np_random)
    return (torch.from_numpy(image), torch.from_numpy(label), torch.tensor(aug, dtype=torch.float64), np.array(image.shape), f["name"])


def cityscapes_id_tables():
    """-> (to_train, to_label): uint8[256] numpy tables label id -> train id (reference datasets.py:146-151, what the training
    loader applies) and train id -> label id (evaluate.py:188, id2trainId(..., reverse=True)), both from the library's one copy."""
    from .. import _cabi
    to_train, to_label = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    _cabi.lib().skd_cityscapes_id_tables(to_train.ctypes.data, to_label.ctypes.data)
    return to_train, to_label


CAMVID_CLASSES = ("Sky", "Building", "Pole", "Road", "Pavement", "Tree", "SignSymbol", "Fence", "Car", "Pedestrian", "Bicyclist")


def camvid_label_table(ignore_label=IGNORE_LABEL):
    """-> uint8[256]: the SegNet CamVid encoding.  Values 0..10 are the classes of `CAMVID_CLASSES` and pass through; every other
    value, 11 (void) included, becomes `ignore_label`."""
    table = np.full(256, ignore_label, np.uint8)
    table[:len(CAMVID_CLASSES)] = np.arange(len(CAMVID_CLASSES), dtype=np.uint8)
    return table


class CamVidDataSet(CSDataSet):
    """CamVid training / validation loader in the SegNet encoding (11 classes, void and every other value ignored).  It is
    `CSDataSet` with another label table: the same list format (`image_path label_path` per line, relative to `root`), the same
    scale rule and random draws (`CS_SCALES`), the same float32 mean, padding, crop and mirror, and `CSDataLoader` yields the same
    `(images, labels, size, name)` batches.  Evaluate with `scale=False, mirror=False` at crop_size=(360, 480)."""

    def __init__(self, root, list_path, max_iters=None, crop_size=(360, 480), mean=(128, 128, 128), scale=True, mirror=True, ignore_label=255):
        super().__init__(root, list_path, max_iters, crop_size, mean, scale, mirror, ignore_label)
        self.label_table = camvid_label_table(ignore_label)


def _label_table_of(dataset):
    """The raw-label -> class table a training loader applies: its own `label_table`, none for VOC, the Cityscapes id table."""
    table = getattr(dataset, "label_table", None)
    if table is not None:
        return table
    if isinstance(dataset, VOCDataSet):
        return np.arange(256, dtype=np.uint8)
    return cityscapes_id_tables()[0]


def class_frequency_weights(dataset, num_classes, c=1.02):
    """-> float32[num_classes] ENet class weights w_k = 1 / ln(c + p_k), p_k = class k's share of the dataset's labelled pixels
    (those whose class, after the loader's label table, is in 0..num_classes-1).  Reads every label file of `dataset` once (a list
    repeated by `max_iters` counts each file once) with no augmentation; a one-off host pass meant for `args.class_weights`."""
    import cv2
    table = _label_table_of(dataset)
    counts = np.zeros(num_classes, np.int64)
    for path in dict.fromkeys(f["label"] for f in dataset.files):
        label = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
        if label is None:
            raise IOError("cannot read %s" % path)
        counts += np.bincount(table[label].ravel(), minlength=256)[:num_classes]
    total = counts.sum()
    if total == 0:
        raise ValueError("no labelled pixel in 0..%d" % (num_classes - 1))
    return (1.0 / np.log(c + counts / total)).astype(np.float32)


class CSDataTestSet(data.Dataset):
    """Same constructor as the reference (datasets.py:213).  `__getitem__` returns the RAW decoded file, its shape and its name:
    (image uint8 H x W x 3 BGR, size int[3], name).  The mean subtraction and padding to crop_size run on the GPU
    (`DeviceTestPreprocess`, through `CSDataLoader`).  Like the reference, it subtracts the BGR ImageNet mean whatever `mean` says."""

    MEAN = (104.00698793, 116.66876762, 122.67891434)       # datasets.py:217

    def __init__(self, root, list_path, crop_size=(505, 505), mean=(128, 128, 128)):
        self.root, self.list_path = root, list_path
        self.crop_h, self.crop_w = crop_size
        self.mean = self.MEAN
        self.img_ids = [i_id.strip().split() for i_id in open(list_path)]
        self.files = [{"img": osp.join(self.root, item[0]), "name": osp.splitext(osp.basename(item[0]))[0]} for item in self.img_ids]

    def __len__(self):
        return len(self.files)

    def __getitem__(self, index):
        import cv2
        f = self.files[index]
        image = cv2.imread(f["img"], cv2.IMREAD_COLOR)
        if image is None:
            raise IOError("cannot read %s" % f["img"])
        return torch.from_numpy(image), np.array(image.shape), f["name"]


def numpy_mean(mean):
    """-> float64[3]: the mean that numpy's `float32 image -= mean` (datasets.py:54, :109) subtracts, exactly.  A float32 array (or a
    Python scalar) is subtracted in float32, i.e. rounded to float32 first; a tuple of Python numbers becomes an int64 / float64
    array and is subtracted in double.  (float)((double)x - m) of this value is numpy's result in both cases."""
    m = -(np.zeros(3, np.float32) - mean)                   # numpy's own promotion; 0 - m is exact in the promoted type
    return np.asarray(m, np.float64).reshape(3)


class VOCDataSet(data.Dataset):
    """Same constructor as the reference (datasets.py:13): `list_path` holds one image name per line, the files are
    `JPEGImages/<name>.jpg` and `SegmentationClassAug/<name>.png` under `root`.  `__getitem__` returns what `CSDataSet`'s does: the RAW
    decoded files and the drawn augmentation (image uint8 H x W x 3 BGR, label uint8 H x W, aug float64[7], size int[3], name).
    Labels are class ids and pass through unchanged; the mean is subtracted on the GPU with numpy's type (`numpy_mean`)."""

    scales = VOC_SCALES

    def __init__(self, root, list_path, max_iters=None, crop_size=(321, 321), mean=(128, 128, 128), scale=True, mirror=True, ignore_label=255):
        self.root, self.list_path = root, list_path
        self.crop_h, self.crop_w = crop_size
        self.scale, self.is_mirror, self.ignore_label = scale, mirror, ignore_label
        self.mean = mean
        self.img_ids = [i_id.strip() for i_id in open(list_path)]
        if max_iters is not None:
            self.img_ids = self.img_ids * int(np.ceil(float(max_iters) / len(self.img_ids)))
        self.files = [{"img": osp.join(self.root, "JPEGImages/%s.jpg" % name), "label": osp.join(self.root, "SegmentationClassAug/%s.png" % name),
                       "name": name} for name in self.img_ids]

    def __len__(self):
        return len(self.files)

    def __getitem__(self, index):
        return _training_sample(self, index)


class VOCDataTestSet(data.Dataset):
    """Same constructor as the reference (datasets.py:85).  `__getitem__` returns the RAW decoded file in the reference's order:
    (image uint8 H x W x 3 BGR, name, size int[3]).  Unlike `CSDataTestSet` it subtracts the `mean` it is given, with numpy's type;
    the subtraction and the zero padding to crop_size run on the GPU (`DeviceTestPreprocess`, through `CSDataLoader`)."""

    def __init__(self, root, list_path, crop_size=(505, 505), mean=(128, 128, 128)):
        self.root, self.list_path = root, list_path
        self.crop_h, self.crop_w = crop_size
        self.mean = mean
        self.img_ids = [i_id.strip() for i_id in open(list_path)]
        self.files = [{"img": osp.join(self.root, "JPEGImages/%s.jpg" % name), "name": name} for name in self.img_ids]

    def __len__(self):
        return len(self.files)

    def __getitem__(self, index):
        import cv2
        f = self.files[index]
        image = cv2.imread(f["img"], cv2.IMREAD_COLOR)
        if image is None:
            raise IOError("cannot read %s" % f["img"])
        return torch.from_numpy(image), osp.splitext(osp.basename(f["img"]))[0], np.array(image.shape)


class DeviceTestPreprocess:
    """raw test images -> float32 [B, 3, max(H, crop_h), max(W, crop_w)] on the device: (float)((double)x - mean[c]) with zero
    padding on the bottom / right and no crop (datasets.py:239-249), one kernel launch per image."""

    def __init__(self, crop_size, mean, device=None):
        from .. import _cabi
        self._lib = _cabi.lib()
        self.crop_h, self.crop_w = crop_size
        self.mean = np.array([float(m) for m in mean], dtype=np.float64)
        self.device = torch.device("cuda") if device is None else torch.device(device)

    def __call__(self, images):
        """images: uint8 [B,H,W,3] tensor or list of [H,W,3] (the batch's padded sizes must agree, as default collation needs)."""
        dev = [t.to(self.device, non_blocking=True).contiguous() for t in images]
        for t in dev:
            if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
                raise ValueError("raw image must be uint8 H x W x 3")
        shapes = {(max(int(t.shape[0]), self.crop_h), max(int(t.shape[1]), self.crop_w)) for t in dev}
        if len(shapes) != 1:
            raise ValueError("test images of one batch pad to different sizes %s: use batch_size=1" % sorted(shapes))
        (oh, ow), = shapes
        out = torch.empty((len(dev), 3, oh, ow), dtype=torch.float32, device=self.device)
        for i, t in enumerate(dev):
            self._lib.skd_cs_test_preprocess(int(t.shape[0]), int(t.shape[1]), t.data_ptr(), self.mean.ctypes.data, oh, ow, out[i].data_ptr(),
                                             torch.cuda.current_stream().cuda_stream)
        self._keep = dev                                                     # raw buffers stay referenced until the next batch
        return out


def _collate_test(batch):
    imgs, sizes, names = zip(*batch)
    same = all(i.shape == imgs[0].shape for i in imgs)
    return torch.stack(imgs) if same else list(imgs), torch.from_numpy(np.stack(sizes)), list(names)


def _collate_voc_test(batch):
    return _collate_test([(image, size, name) for image, name, size in batch])


class _Sample(ctypes.Structure):          # include/skd.h: skd_cs_sample
    _fields_ = [("image", ctypes.c_void_p), ("label", ctypes.c_void_p), ("src_h", ctypes.c_int), ("src_w", ctypes.c_int),
                ("f_scale", ctypes.c_double), ("scaled_h", ctypes.c_int), ("scaled_w", ctypes.c_int), ("h_off", ctypes.c_int),
                ("w_off", ctypes.c_int), ("flip", ctypes.c_int)]


class DeviceAugment:
    """raw batch -> (images float32 [B,3,crop_h,crop_w], labels [B,crop_h,crop_w]) on the device, one kernel launch.

    `label_dtype`: torch.float32 is what the reference's `__getitem__` returns; torch.int64 is what `NetModel.set_input` makes of it
    (`labels.long()`, kd_model.py:105) -- the default, it saves that conversion pass.
    `voc`: False (Cityscapes) maps label ids to train ids and subtracts the mean rounded to float32; True (PASCAL VOC) passes labels
    through and subtracts the mean with numpy's type (`numpy_mean`).
    `table`: with voc=False, a uint8[256] raw label -> class table to apply instead of the Cityscapes one (`camvid_label_table`)."""

    def __init__(self, crop_size, mean, ignore_label=IGNORE_LABEL, label_dtype=torch.int64, device=None, voc=False, table=None):
        from .. import _cabi
        self._lib = _cabi.lib()
        self.crop_h, self.crop_w = crop_size
        if voc:
            if table is not None:
                raise ValueError("a VOC loader applies no label table")
            self.mean, self.table = numpy_mean(mean), None
        else:
            if table is None:
                table = cityscapes_id_tables()[0]
            table = np.ascontiguousarray(table, np.uint8)
            if table.shape != (256,):
                raise ValueError("label table must have 256 entries (got shape %s)" % (table.shape,))
            self.mean, self.table = np.array([np.float32(m) for m in mean], np.float64), table
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
        self._lib.skd_augment_batch(n, ctypes.cast(arr, ctypes.c_void_p), self.crop_h, self.crop_w, self.mean.ctypes.data,
                                    None if self.table is None else self.table.ctypes.data, self.ignore_label, out_i.data_ptr(),
                                    out_l.data_ptr(), 1 if self.label_dtype == torch.int64 else 0, torch.cuda.current_stream().cuda_stream)
        self._keep = (dev_i, dev_l)                                          # raw buffers stay referenced until the next batch
        return out_i, out_l


def _collate(batch):
    """default collate, except that raw files of different sizes stay lists"""
    imgs, labs, augs, sizes, names = zip(*batch)
    same = all(i.shape == imgs[0].shape for i in imgs)
    return (torch.stack(imgs) if same else list(imgs), torch.stack(labs) if same else list(labs), torch.stack(augs),
            torch.from_numpy(np.stack(sizes)), list(names))


class _ReplayDraws:
    """worker_init_fn of a resumed iteration: worker `w` makes, without reading the files, the `draw_augmentation` calls it made for
    the batches it loaded before batch `start` of the interrupted iteration (batches go to the workers round-robin: batch b to worker
    b % num_workers), so its `random` / `np.random` continue where they were.  Image sizes come from the file headers (`image_size`),
    once per distinct file."""

    def __init__(self, dataset, order, batch_size, start, num_workers):
        self.dataset, self.order, self.batch_size, self.start, self.num_workers = dataset, order, batch_size, start, num_workers

    def __call__(self, worker_id):
        ds, sizes = self.dataset, {}
        for b in range(worker_id, self.start, self.num_workers):
            for index in self.order[b * self.batch_size:(b + 1) * self.batch_size]:
                path = ds.files[index]["img"]
                if path not in sizes:
                    sizes[path] = image_size(path)
                h, w = sizes[path]
                draw_augmentation(h, w, (ds.crop_h, ds.crop_w), ds.scale, ds.is_mirror, ds.scales)


class _KeyedSamples(data.Dataset):
    """The dataset as a partitioned loader reads it: item (index, iteration, position) -> sample `index`, its augmentation drawn from
    `keyed_generators(seed, iteration, position)`; a test split makes no draws."""

    def __init__(self, dataset, seed, test):
        self.dataset, self.seed, self.test = dataset, seed, test

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, item):
        index, iteration, position = item
        if self.test:
            return self.dataset[index]
        return _training_sample(self.dataset, index, *keyed_generators(self.seed, iteration, position))


class CSDataLoader:
    """Drop-in for `data.DataLoader(CSDataSet(...), batch_size=..., shuffle=True, num_workers=4, pin_memory=True)` of
    train_and_eval.py:13-15: iterating it yields `(images, labels, size, name)` with images / labels already augmented and on the GPU,
    for a `CSDataSet` or a `VOCDataSet`.  With a `CSDataTestSet` (test.py:9-10) it yields `(images, size, name)`, with a
    `VOCDataTestSet` `(images, name, size)` (the reference's orders), images mean-subtracted and padded on the GPU.

    A training loader can be resumed: `state_dict()` is the position of the current iteration, and after `load_state_dict(sd)` the
    next iteration yields the batches that iteration had not yet yielded -- the same samples in the same order with the same
    augmentation draws.  With num_workers > 0 the workers' draws are replayed; with num_workers == 0 they come from this process's
    `random` / `np.random`, which must be restored too (`StepModel.load_training_state` does both).  Without a loaded position every
    iteration is torch's DataLoader's, unchanged.

    Data parallel: with `rank` and `world_size` (e.g. `dist.get_rank()`, `dist.get_world_size()`) the loader yields this rank's share
    of one order common to all ranks.  Iteration e (counted from 0 over the calls to `__iter__` / `host_batches`) takes the order
    `partition_order(len(dataset), seed, e, shuffle)`; global batch g is its positions [g*W*b, (g+1)*W*b) and rank r yields
    [g*W*b + r*b, g*W*b + (r+1)*b) of them (W = world_size, b = batch_size).  A partial last global batch is dropped on every rank
    with `drop_last=True` (all ranks yield len(self) batches), and shared out in rank order otherwise (a rank may get a short batch
    or none: with b = 1 and no shuffle rank r gets samples r, r + W, ...).  The augmentation of the sample at global position p is
    drawn from `keyed_generators(seed, e, p)`: rank, worker count and resume point do not change it, and the process's `random`,
    `np.random` and torch streams are not used.  So the W ranks' batch g, concatenated in rank order, is batch g of a
    `world_size=1, batch_size=W*b` loader with the same seed.  `seed` means nothing without `rank` / `world_size`."""

    def __init__(self, dataset, batch_size=1, shuffle=False, num_workers=0, pin_memory=True, drop_last=False, label_dtype=torch.int64,
                 device=None, rank=None, world_size=None, seed=0):
        if (rank is None) != (world_size is None):
            raise ValueError("rank and world_size are given together (got rank=%r, world_size=%r)" % (rank, world_size))
        if world_size is not None:
            ints = all(isinstance(v, int) and not isinstance(v, bool) for v in (rank, world_size, seed))
            if not ints or world_size < 1 or not 0 <= rank < world_size or seed < 0:
                raise ValueError("a partitioned loader needs integers 0 <= rank < world_size and seed >= 0 (got rank=%r, world_size=%r, "
                                 "seed=%r)" % (rank, world_size, seed))
        self.rank, self.world_size, self.seed = rank, world_size, seed
        self._iteration, self._current = 0, None          # partitioned: the next iteration's index, the current (or last) one's
        self.dataset = dataset
        self.voc = isinstance(dataset, (VOCDataSet, VOCDataTestSet))
        self.test = isinstance(dataset, (CSDataTestSet, VOCDataTestSet))
        collate = (_collate_voc_test if self.voc else _collate_test) if self.test else _collate
        self.loader = data.DataLoader(dataset, batch_size=batch_size, shuffle=shuffle, num_workers=num_workers, pin_memory=pin_memory,
                                      drop_last=drop_last, collate_fn=collate)
        if self.test:
            mean = numpy_mean(dataset.mean) if self.voc else dataset.mean
            self.augment = DeviceTestPreprocess((dataset.crop_h, dataset.crop_w), mean, device)
        else:
            self.augment = DeviceAugment((dataset.crop_h, dataset.crop_w), dataset.mean, dataset.ignore_label, label_dtype, device, self.voc,
                                         getattr(dataset, "label_table", None))
        self._shuffle = shuffle
        self._iter_rng, self._yielded, self._resume = None, 0, None

    def __len__(self):
        if self.world_size is None:
            return len(self.loader)
        n, b, step = len(self.dataset), self.loader.batch_size, self.world_size * self.loader.batch_size
        full = n // step
        return full if self.loader.drop_last else full + int(n - full * step > self.rank * b)

    def __iter__(self):
        if self.test:
            for images, sizes, names in (self.loader if self.world_size is None else self._partitioned()):
                yield (self.augment(images), names, sizes) if self.voc else (self.augment(images), sizes, names)
            return
        for images, labels, augs, sizes, names in self.host_batches():
            out_i, out_l = self.augment(images, labels, augs)
            yield out_i, out_l, sizes, names

    # ---- resuming ---------------------------------------------------------------------------------------------------------------
    def host_batches(self):
        """One iteration's raw training batches `(images, labels, augs, sizes, names)` as the workers return them, before the device
        step (what `__iter__` augments): the rest of an interrupted iteration after `load_state_dict`, else a whole new one."""
        if self.test:
            raise ValueError("only a training loader (CSDataSet / VOCDataSet) yields augmentation batches")
        if self.world_size is not None:
            yield from self._partitioned()
            return
        resume, self._resume = self._resume, None
        if resume is None:
            # torch's iterator draws the workers' base seed and then the sampler's seed from the default generator: its state here
            # fixes both
            self._iter_rng, self._yielded = torch.get_rng_state(), 0
            it, skip = iter(self.loader), 0
        else:
            self._iter_rng, self._yielded = resume
            it, skip = self._resumed(*resume)
        for batch in it:
            if skip:
                skip -= 1
                continue
            self._yielded += 1
            yield batch

    def _resumed(self, rng, start):
        """-> (iterator, batches to drop): torch's iterator of the interrupted iteration, rebuilt from the default generator's state
        `rng` at its start, beginning at the first batch >= start - num_workers + 1 whose worker is the one that loaded it then."""
        n, bs, workers = len(self.dataset), self.loader.batch_size, self.loader.num_workers
        g = torch.Generator()
        g.set_state(rng)
        torch.empty((), dtype=torch.int64).random_(generator=g)              # the workers' base seed
        order = list(range(n))
        if self._shuffle:                                                    # RandomSampler: a seed, then randperm from it
            seed = int(torch.empty((), dtype=torch.int64).random_(generator=g).item())
            order = torch.randperm(n, generator=torch.Generator().manual_seed(seed)).tolist()
        first = start - start % workers if workers else start
        base = torch.Generator()
        base.set_state(rng)                                                  # the DataLoader draws the same base seed from it
        loader = data.DataLoader(self.dataset, batch_size=bs, sampler=order[first * bs:], num_workers=workers,
                                 pin_memory=self.loader.pin_memory, drop_last=self.loader.drop_last, collate_fn=self.loader.collate_fn,
                                 generator=base, worker_init_fn=_ReplayDraws(self.dataset, order, bs, first, workers) if first else None)
        return iter(loader), start - first

    def _rank_batches(self, iteration):
        """-> this rank's batches of partitioned iteration `iteration`, each a list of (dataset index, iteration, global position)."""
        n, b, step = len(self.dataset), self.loader.batch_size, self.world_size * self.loader.batch_size
        order = partition_order(n, self.seed, iteration, self._shuffle)
        stop = n - n % step if self.loader.drop_last else n
        return [[(order[p], iteration, p) for p in range(start, min(start + b, stop))] for start in range(self.rank * b, stop, step)]

    def _partitioned(self):
        """One partitioned iteration's raw batches: the rest of an interrupted one after `load_state_dict`, else the next one."""
        resume, self._resume = self._resume, None
        iteration, start = (self._iteration, 0) if resume is None else resume
        self._iteration, self._current, self._yielded = iteration + 1, iteration, start
        batches = self._rank_batches(iteration)[start:]
        if not batches:
            return
        # a private generator for the workers' base seed, so that the default one is left alone
        loader = data.DataLoader(_KeyedSamples(self.dataset, self.seed, self.test), batch_sampler=batches,
                                 num_workers=self.loader.num_workers, pin_memory=self.loader.pin_memory, collate_fn=self.loader.collate_fn,
                                 generator=torch.Generator())
        for batch in loader:
            self._yielded += 1
            yield batch

    def state_dict(self):
        """The position of the current (or last) iteration: the default generator's state when it began, and the number of batches
        it has yielded.  A partitioned loader (version 2) holds its iteration index instead of a generator state, with its `rank`,
        `world_size`, `seed` and `drop_last`."""
        if self.test:
            raise ValueError("only a training loader (CSDataSet / VOCDataSet) can be resumed")
        sd = dict(version=1, rng_state=self._iter_rng, batches=self._yielded, num_samples=len(self.dataset),
                  batch_size=self.loader.batch_size, shuffle=self._shuffle, num_workers=self.loader.num_workers)
        if self.world_size is not None:
            sd.update(version=2, rng_state=None, rank=self.rank, world_size=self.world_size, seed=self.seed, iteration=self._current,
                      drop_last=self.loader.drop_last)
        return sd

    def load_state_dict(self, sd):
        """The next iteration continues the one `sd` describes (state_dict of a loader over the same list, batch size, shuffle and
        worker count, and for a partitioned loader the same rank, world size, seed and drop_last); a mismatch raises ValueError naming
        the field, and changes nothing."""
        if self.test:
            raise ValueError("only a training loader (CSDataSet / VOCDataSet) can be resumed")
        want = dict(rank=self.rank, world_size=self.world_size)
        if self.world_size is not None:
            want.update(seed=self.seed, drop_last=self.loader.drop_last)
        want.update(version=1 if self.world_size is None else 2, num_samples=len(self.dataset), batch_size=self.loader.batch_size,
                    shuffle=self._shuffle, num_workers=self.loader.num_workers)
        for k, v in want.items():
            if sd.get(k) != v:
                raise ValueError("loader state does not match the loader: %s is %r, the loader's %r" % (k, sd.get(k), v))
        if self.world_size is not None:                                      # iteration None: none had begun, start at the first
            self._resume = (0, 0) if sd["iteration"] is None else (int(sd["iteration"]), int(sd["batches"]))
        elif sd["rng_state"] is not None:                                    # None: no iteration had begun, nothing to skip
            self._resume = (sd["rng_state"].clone(), int(sd["batches"]))
