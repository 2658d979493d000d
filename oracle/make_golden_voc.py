"""TEST INFRASTRUCTURE -- generates tests/golden/voc_dataset.pt.gz by running the UNMODIFIED reference PASCAL VOC loaders.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_voc        (needs cv2)

Writes synthetic VOC-layout files (`JPEGImages/<name>.jpg`, `SegmentationClassAug/<name>.png`: uint8 BGR images, class ids 0..20
plus some 255) to a temporary directory, points the reference's `dataset/datasets.py::VOCDataSet` and `VOCDataTestSet` (imported as
shipped, through oracle/make_golden_dataset.py's loader) at them, seeds `random` / `np.random`, and records for every case: the
arrays as cv2.imread decodes the files (JPEG is lossy: these, not the arrays before encoding, are the loader's input), the
constructor arguments, the seeds and what the reference returned.  oracle/voc_port.py is held to these bit for bit
(tests/test_voc_cpu.py), and the CUDA kernels to both (tests/test_voc_gpu.py).
"""
import gzip
import io
import os
import random
import tempfile

import numpy as np
import torch

from .make_golden_dataset import IMG_MEAN, load_reference_dataset_module
from .voc_port import voc_getitem

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "voc_dataset.pt.gz")
TUPLE_MEAN = (104.00698793, 116.66876762, 122.67891434)          # Python floats: the reference subtracts them in double

# (name, raw H, raw W, crop (h, w), scale, mirror, number of draws, mean)
CASES = [
    ("train_all_scales", 60, 80, (33, 45), True, True, 24, IMG_MEAN),         # seed chosen so that all 12 scale indices show up
    ("train_odd_sizes_tuple_mean", 37, 53, (41, 47), True, True, 10, TUPLE_MEAN),
    ("train_default_mean", 45, 61, (33, 33), True, True, 6, (128, 128, 128)),
    ("train_no_aug", 40, 72, (32, 64), False, False, 3, TUPLE_MEAN),
    ("train_mirror_only", 40, 72, (40, 72), False, True, 4, IMG_MEAN),
    ("val_padded", 30, 50, (32, 64), False, False, 2, TUPLE_MEAN),           # evaluation: scale=False, mirror=False, pads
]
# (name, raw H, raw W, crop (h, w), mean)
TEST_CASES = [
    ("test_smaller", 30, 41, (40, 48), TUPLE_MEAN),
    ("test_larger", 50, 70, (40, 48), IMG_MEAN),
    ("test_across", 30, 70, (40, 48), (128, 128, 128)),
]


def _synthetic(rng, H, W):
    yy, xx = np.mgrid[0:H, 0:W]
    base = (np.stack([xx * 3 + yy, yy * 5, (xx + yy) * 2], -1) % 256).astype(np.int64)
    img = ((base + rng.integers(0, 64, (H, W, 3))) % 256).astype(np.uint8)
    lab = rng.integers(0, 21, (H, W)).astype(np.uint8)
    lab[rng.random((H, W)) < 0.05] = 255
    lab = np.repeat(np.repeat(lab[::4, ::4], 4, 0), 4, 1)[:H, :W].copy()
    return img, lab


def _draw_all(ds, seed, draws):
    random.seed(seed); np.random.seed(seed)
    return [ds[0] for _ in range(draws)]


def main():
    import cv2
    ref = load_reference_dataset_module()
    rng = np.random.default_rng(4321)
    out = {"cv2": cv2.__version__, "cases": [], "test_cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "JPEGImages")); os.makedirs(os.path.join(tmp, "SegmentationClassAug"))
        for ci, (name, H, W, crop, scale, mirror, draws, mean) in enumerate(CASES):
            img, lab = _synthetic(rng, H, W)
            stem = "2007_%06d" % ci
            ip, lp = os.path.join(tmp, "JPEGImages", stem + ".jpg"), os.path.join(tmp, "SegmentationClassAug", stem + ".png")
            assert cv2.imwrite(ip, img) and cv2.imwrite(lp, lab)
            lst = os.path.join(tmp, "list%d.txt" % ci)
            with open(lst, "w") as f:
                f.write(stem + "\n")
            ds = ref.VOCDataSet(tmp, lst, crop_size=crop, mean=mean, scale=scale, mirror=mirror)
            seed = 200 + ci
            if name == "train_all_scales":
                # first seed whose draws cover the 12 scale indices, found with oracle/voc_port.py's draws on the decoded files (the
                # test then holds the reference's outputs at that seed to the port's, which pins the coverage)
                dec_i, dec_l = cv2.imread(ip, cv2.IMREAD_COLOR), cv2.imread(lp, cv2.IMREAD_GRAYSCALE)
                while True:
                    random.seed(seed); np.random.seed(seed)
                    ks = {voc_getitem(dec_i, dec_l, crop, mean, scale, mirror)[2]["scale_idx"] for _ in range(draws)}
                    if len(ks) == 12:
                        break
                    seed += 1
            items = []
            for image, label, size, nm in _draw_all(ds, seed, draws):
                assert nm == stem
                items.append((torch.from_numpy(image), torch.from_numpy(label)))
            out["cases"].append({"name": name, "stem": stem, "raw_image": torch.from_numpy(cv2.imread(ip, cv2.IMREAD_COLOR)),
                                 "raw_label": torch.from_numpy(cv2.imread(lp, cv2.IMREAD_GRAYSCALE)), "crop": crop, "scale": scale,
                                 "mirror": mirror, "mean": mean, "seed": seed, "items": items, "size": tuple(int(v) for v in size)})
            print(name, "seed", seed, "draws", draws, "image", tuple(items[0][0].shape))
        for ci, (name, H, W, crop, mean) in enumerate(TEST_CASES):
            img, _ = _synthetic(rng, H, W)
            stem = "2008_%06d" % ci
            ip = os.path.join(tmp, "JPEGImages", stem + ".jpg")
            assert cv2.imwrite(ip, img)
            lst = os.path.join(tmp, "test%d.txt" % ci)
            with open(lst, "w") as f:
                f.write(stem + "\n")
            image, nm, size = ref.VOCDataTestSet(tmp, lst, crop_size=crop, mean=mean)[0]
            assert nm == stem
            out["test_cases"].append({"name": name, "stem": stem, "raw_image": torch.from_numpy(cv2.imread(ip, cv2.IMREAD_COLOR)),
                                      "crop": crop, "mean": mean, "image": torch.from_numpy(np.ascontiguousarray(image)),
                                      "size": tuple(int(v) for v in size)})
            print(name, "image", tuple(image.shape), image.dtype)
        # constructors only: the file layout and the max_iters repetition
        lst = os.path.join(tmp, "names.txt")
        with open(lst, "w") as f:
            f.write("2007_000032\n2007_000039\n2008_000123\n")
        tr, te = ref.VOCDataSet(tmp, lst, max_iters=7), ref.VOCDataTestSet(tmp, lst)
        rel = lambda p: os.path.relpath(p, tmp)
        out["layout"] = {"train": [(rel(f["img"]), rel(f["label"]), f["name"]) for f in tr.files],
                         "test": [rel(f["img"]) for f in te.files], "max_iters": 7}
    buf = io.BytesIO(); torch.save(out, buf)
    with open(OUT, "wb") as f:
        f.write(gzip.compress(buf.getvalue(), 9, mtime=0))
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KB")


if __name__ == "__main__":
    main()
