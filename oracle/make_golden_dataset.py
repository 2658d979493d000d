"""TEST INFRASTRUCTURE -- generates tests/golden/dataset.pt.gz by running the UNMODIFIED reference loader.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_dataset        (needs cv2)

Writes synthetic Cityscapes-like PNG pairs (uint8 BGR image, uint8 label ids 0..33 plus some 255) to a temporary directory, points the
reference's `dataset/datasets.py::CSDataSet` (imported as shipped; only `torchvision`, which it imports and never uses, is stubbed when
absent) at them, seeds `random` / `np.random`, and records for every case: the raw arrays, the constructor arguments, the seeds and
the (image, label) the reference returned.  oracle/dataset_port.py is then held to these bit for bit (tests/test_dataset_cpu.py), and
the CUDA kernel to both (tests/test_dataset_gpu.py).
"""
import gzip
import importlib.util
import io
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

from .refshim import REFERENCE_ROOT

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "dataset.pt.gz")
IMG_MEAN = np.array((104.00698793, 116.66876762, 122.67891434), dtype=np.float32)        # train_and_eval.py:10

# (name, raw H, raw W, crop (h, w), scale, mirror, number of draws)
CASES = [
    ("train_scale_mirror", 64, 128, (48, 80), True, True, 16),        # every scale index shows up; scales < 1 need padding
    ("train_odd_sizes", 37, 53, (41, 47), True, True, 8),
    ("train_no_aug", 40, 72, (32, 64), False, False, 3),
    ("train_mirror_only", 40, 72, (40, 72), False, True, 4),
    ("val_full_image", 32, 64, (32, 64), False, False, 2),             # train_and_eval.py:16: crop = image size, no augmentation
    ("val_padded", 30, 50, (32, 64), False, False, 2),
]


def load_reference_dataset_module():
    if "torchvision" not in sys.modules:
        try:
            import torchvision  # noqa: F401
        except Exception:
            sys.modules["torchvision"] = types.ModuleType("torchvision")
    spec = importlib.util.spec_from_file_location("_ref_datasets", os.path.join(REFERENCE_ROOT, "dataset", "datasets.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import cv2
    ref = load_reference_dataset_module()
    rng = np.random.default_rng(1234)
    out = {"cv2": cv2.__version__, "mean": torch.from_numpy(IMG_MEAN.copy()), "cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        for ci, (name, H, W, crop, scale, mirror, draws) in enumerate(CASES):
            # smooth-ish image content + noise so that interpolation is exercised on gradients and on edges
            yy, xx = np.mgrid[0:H, 0:W]
            base = (np.stack([xx * 3 + yy, yy * 5, (xx + yy) * 2], -1) % 256).astype(np.int64)
            img = ((base + rng.integers(0, 64, (H, W, 3))) % 256).astype(np.uint8)
            lab = rng.integers(0, 34, (H, W)).astype(np.uint8)
            lab[rng.random((H, W)) < 0.03] = 255
            lab = np.repeat(np.repeat(lab[::4, ::4], 4, 0), 4, 1)[:H, :W].copy()       # blocks: nearest-neighbour picks are visible
            ip, lp = os.path.join(tmp, "img%d.png" % ci), os.path.join(tmp, "lab%d.png" % ci)
            assert cv2.imwrite(ip, img) and cv2.imwrite(lp, lab)
            lst = os.path.join(tmp, "list%d.lst" % ci)
            with open(lst, "w") as f:
                f.write("img%d.png lab%d.png\n" % (ci, ci))
            ds = ref.CSDataSet(tmp, lst, crop_size=crop, mean=IMG_MEAN, scale=scale, mirror=mirror)
            seed = 100 + ci
            random.seed(seed); np.random.seed(seed)
            items = []
            for _ in range(draws):
                image, label, size, nm = ds[0]
                items.append((torch.from_numpy(image), torch.from_numpy(label)))
            out["cases"].append({"name": name, "raw_image": torch.from_numpy(img), "raw_label": torch.from_numpy(lab), "crop": crop,
                                 "scale": scale, "mirror": mirror, "seed": seed, "items": items, "size": tuple(int(v) for v in size)})
            print(name, "draws", draws, "image", tuple(items[0][0].shape), "label", tuple(items[0][1].shape))
    buf = io.BytesIO(); torch.save(out, buf)
    with open(OUT, "wb") as f:                                  # gzip: the u8-derived values compress ~3x (fixtures stay < 1 MB)
        f.write(gzip.compress(buf.getvalue(), 9, mtime=0))
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KB")


if __name__ == "__main__":
    main()
