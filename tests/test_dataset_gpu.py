"""GPU: `skd_cs_augment_batch` (csrc/augment.cu) through `DeviceAugment` / `CSDataLoader` against (1) the outputs of the UNMODIFIED
reference loader stored in tests/golden/dataset.pt.gz and (2) the oracle restatement on seeded full-size inputs (1024 x 2048 -> 512 x 1024,
all 15 scale factors).  Integer / table work and one float32 subtraction: the bar is bit-exact."""
import gzip
import os
import random

import numpy as np
import pytest
import torch

from oracle import dataset_port as dp

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "dataset.pt.gz")


def _augs(img, crop, scale, mirror, n):
    from structure_knowledge_distillation_b200.dataset.datasets import draw_augmentation
    return [draw_augmentation(img.shape[0], img.shape[1], crop, scale, mirror) for _ in range(n)]


def test_device_augment_matches_reference_loader_golden():
    from structure_knowledge_distillation_b200.dataset.datasets import DeviceAugment
    gold = torch.load(gzip.open(GOLD), weights_only=False)
    mean = gold["mean"].numpy()
    total = 0
    for case in gold["cases"]:
        img, lab = case["raw_image"], case["raw_label"]
        n = len(case["items"])
        random.seed(case["seed"]); np.random.seed(case["seed"])
        augs = _augs(img, case["crop"], case["scale"], case["mirror"], n)
        for dtype in (torch.float32, torch.int64):
            aug = DeviceAugment(case["crop"], mean, 255, label_dtype=dtype)
            out_i, out_l = aug([img] * n, [lab] * n, torch.tensor(augs, dtype=torch.float64))
            torch.cuda.synchronize()
            for k, (ri, rl) in enumerate(case["items"]):
                assert torch.equal(out_i[k].cpu(), ri), (case["name"], k)
                assert torch.equal(out_l[k].cpu().float(), rl), (case["name"], k)
                total += 1
    print("PARITY dataset_golden %d samples bit-exact vs the reference CSDataSet (cv2 %s)" % (total // 2, gold["cv2"]))


def test_device_augment_full_size_all_scales_vs_oracle():
    from structure_knowledge_distillation_b200.dataset.datasets import DeviceAugment, Augmentation
    rng = np.random.default_rng(7)
    H, W, crop = 1024, 2048, (512, 1024)
    mean = np.array((104.00698793, 116.66876762, 122.67891434), dtype=np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    img = ((np.stack([xx + yy, 2 * yy, 3 * xx], -1) + rng.integers(0, 96, (H, W, 3))) % 256).astype(np.uint8)
    lab = rng.integers(0, 34, (H // 8, W // 8)).astype(np.uint8).repeat(8, 0).repeat(8, 1)
    lab[rng.random((H, W)) < 0.01] = 255
    augs, want = [], []
    for k in range(15):

        class _Fixed:                                            # the oracle draws what we tell it to: scale index k first
            def __init__(self): self.calls = 0
            def randint(self, a, b):
                self.calls += 1
                return k if self.calls == 1 else int(rng.integers(a, b + 1))
        class _Flip:
            @staticmethod
            def choice(n): return int(rng.integers(0, n))
        wi, wl, p = dp.cs_getitem(img, lab, crop, mean, scale=True, mirror=True, py_random=_Fixed(), np_random=_Flip)
        f = p["f_scale"]
        augs.append(Augmentation(k, f, dp.cv_round(H * f), dp.cv_round(W * f), p["h_off"], p["w_off"], p["flip"]))
        want.append((wi, wl))
    aug = DeviceAugment(crop, mean, 255, label_dtype=torch.int64)
    ti, tl = torch.from_numpy(img), torch.from_numpy(lab)
    out_i, out_l = aug(torch.stack([ti] * 15), torch.stack([tl] * 15), torch.tensor(augs, dtype=torch.float64))
    torch.cuda.synchronize()
    for k in range(15):
        assert np.array_equal(out_i[k].cpu().numpy(), want[k][0]), k
        assert np.array_equal(out_l[k].cpu().numpy().astype(np.float32), want[k][1]), k
    # throughput of the kernel alone (reported, not asserted)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    di, dl = torch.stack([ti] * 8).cuda(), torch.stack([tl] * 8).cuda()
    a8 = torch.tensor(augs[:8], dtype=torch.float64)
    for _ in range(3):
        aug(di, dl, a8)
    e0.record()
    for _ in range(10):
        aug(di, dl, a8)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("PARITY dataset_full_size 15 scale factors bit-exact vs oracle; batch 8 of 512x1024 crops from 1024x2048 files: %.3f ms "
          "(%.0f images/s, %.0f GB/s of output)" % (ms, 8 / ms * 1e3, 8 * 512 * 1024 * (12 + 8) / ms / 1e6))


def test_loader_end_to_end_into_set_input(tmp_path):
    """files -> CSDataLoader -> device batch with the shapes / dtypes `NetModel.set_input` takes, same draws as a seeded oracle."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataSet, CSDataLoader
    rng = np.random.default_rng(3)
    mean = np.array((104.00698793, 116.66876762, 122.67891434), dtype=np.float32)
    raws = []
    with open(tmp_path / "train.lst", "w") as f:
        for i in range(4):
            img = rng.integers(0, 256, (96, 160, 3), dtype=np.uint8); lab = rng.integers(0, 34, (96, 160), dtype=np.uint8)
            cv2.imwrite(str(tmp_path / ("i%d.png" % i)), img); cv2.imwrite(str(tmp_path / ("l%d.png" % i)), lab)
            f.write("i%d.png l%d.png\n" % (i, i)); raws.append((img, lab))
    ds = CSDataSet(str(tmp_path), str(tmp_path / "train.lst"), crop_size=(64, 128), mean=mean, scale=True, mirror=True)
    random.seed(5); np.random.seed(5)
    batches = list(CSDataLoader(ds, batch_size=2, shuffle=False, num_workers=0))
    random.seed(5); np.random.seed(5)
    k = 0
    for images, labels, sizes, names in batches:
        assert images.is_cuda and images.dtype == torch.float32 and tuple(images.shape) == (2, 3, 64, 128)
        assert labels.is_cuda and labels.dtype == torch.int64 and tuple(labels.shape) == (2, 64, 128)
        for j in range(2):
            wi, wl, _ = dp.cs_getitem(raws[k][0], raws[k][1], (64, 128), mean, scale=True, mirror=True)
            assert np.array_equal(images[j].cpu().numpy(), wi) and np.array_equal(labels[j].cpu().numpy().astype(np.float32), wl)
            assert names[j] == "l%d" % k and tuple(int(v) for v in sizes[j]) == (96, 160, 3)
            k += 1
    assert k == 4
