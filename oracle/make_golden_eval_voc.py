"""TEST INFRASTRUCTURE -- generates tests/golden/eval_voc.pt.gz by running the UNMODIFIED reference sliding-window evaluation at 21
classes over the unmodified reference `VOCDataSet`, on CPU.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_eval_voc        (needs cv2 and PIL)

Synthetic VOC val files (`JPEGImages/<name>.jpg`, `SegmentationClassAug/<name>.png`) go to a temporary directory.  The reference's
`VOCDataSet(..., crop_size=(512, 512), scale=False, mirror=False, mean=IMG_MEAN)` in a `DataLoader` feeds the reference's
`evaluate_main(net, loader, '0', '512,512', 21, False)` -- the validation configuration of train_and_eval.py with VOC's lists --
with oracle/make_golden_eval.py's fixed-weight `ToyNet(21)` and its call-time CPU / numpy 2 shims.

One more call-time adaptation, for images smaller than the crop (every VOC image: at most 500 pixels a side).  evaluate_main crops the
label to the batch's `size` (the raw image's shape) but not the prediction, and indexes the 512 x 512 prediction with the cropped
mask (evaluate.py:196-199).  numpy 1 read such a mismatched boolean index at the mask's own coordinates, i.e. it counted the prediction
over the image's region; numpy 2 raises IndexError.  The loader is therefore wrapped to report the padded label's shape as `size`: the
padding's labels are all ignore_label, so the confusion counts are what numpy 1 computed.  Images and labels pass unchanged.

Recorded: the files' bytes, the loader's arguments and seed, the reference's mean IU and IU array, its PNGs (the arg-max of each
512 x 512 batch image) and the pixels whose top-2 score margin is below 1e-4.
"""
import gzip
import io
import os
import random
import tempfile

import numpy as np
import torch

from .make_golden_dataset import IMG_MEAN
from .make_golden_eval import TIE, ToyNet, cpu_numpy2_shims, load_reference_eval, raw_image, read_pngs, top2_margin

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "eval_voc.pt.gz")
CLASSES = 21
CROP = (512, 512)
SEED = 31
# (name, H, W): portrait and landscape VOC sizes (padded to the crop), and one larger than the crop (a random 512 x 512 crop)
IMAGES = (("2007_000033", 375, 500), ("2007_000042", 500, 375), ("2007_000061", 530, 560))


def synth_label(H, W, seed):
    """class ids 0..20 in 16-pixel blocks, a 5 % sprinkle of ignore_label and an ignore_label border, as VOC's object outlines"""
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, CLASSES, (H // 16 + 1, W // 16 + 1)).repeat(16, 0).repeat(16, 1)[:H, :W].astype(np.uint8)
    lab[rng.random((H, W)) < 0.05] = 255
    lab[:3] = 255; lab[:, :3] = 255
    return lab


def write_files(root):
    """-> {name: (jpg bytes, png bytes)} written under `root`, plus root/val.txt"""
    import cv2
    os.makedirs(os.path.join(root, "JPEGImages"), exist_ok=True)
    os.makedirs(os.path.join(root, "SegmentationClassAug"), exist_ok=True)
    files = {}
    for i, (name, H, W) in enumerate(IMAGES):
        ip, lp = os.path.join(root, "JPEGImages", name + ".jpg"), os.path.join(root, "SegmentationClassAug", name + ".png")
        assert cv2.imwrite(ip, raw_image(H, W, 50 + i)) and cv2.imwrite(lp, synth_label(H, W, 60 + i))
        files[name] = (open(ip, "rb").read(), open(lp, "rb").read())
    with open(os.path.join(root, "val.txt"), "w") as f:
        f.write("".join(name + "\n" for name, _, _ in IMAGES))
    return files


class PaddedSize:
    """the reference loader with `size` = the (padded) label's shape; see the module docstring"""

    def __init__(self, loader):
        self.loader = loader

    def __iter__(self):
        for image, label, size, name in self.loader:
            yield image, label, torch.tensor([[label.shape[1], label.shape[2], 3]]), name


def main():
    from torch.utils import data
    ev, ds = load_reference_eval()
    torch.set_num_threads(os.cpu_count())
    net = ToyNet(CLASSES).eval()
    cwd = os.getcwd()
    with cpu_numpy2_shims(ev), torch.no_grad(), tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "voc")
        files = write_files(root)

        def loader():
            random.seed(SEED); np.random.seed(SEED)                  # the crop offsets of images larger than the crop
            return data.DataLoader(ds.VOCDataSet(root, os.path.join(root, "val.txt"), crop_size=CROP, mean=IMG_MEAN, scale=False,
                                                 mirror=False), batch_size=1, shuffle=False, pin_memory=False)
        os.makedirs(os.path.join(tmp, "run")); os.chdir(os.path.join(tmp, "run"))
        try:
            miou, iu = ev.evaluate_main(net, PaddedSize(loader()), "0", "%d,%d" % CROP, CLASSES, False, type="val")
            pngs = read_pngs("outputs")
        finally:
            os.chdir(cwd)
        for image, _, size, name in loader():
            scores = ev.predict_sliding(net, image.numpy(), CROP, CLASSES, False, 1)
            pngs[name[0]]["near_ties"] = torch.from_numpy(np.flatnonzero(top2_margin(scores) < TIE))
            pngs[name[0]]["size"] = tuple(int(v) for v in size[0])
            print(name[0], "size", pngs[name[0]]["size"], "near ties", len(pngs[name[0]]["near_ties"]))
    out = dict(classes=CLASSES, crop=CROP, seed=SEED, tie=TIE, mean=IMG_MEAN, images=IMAGES, files=files, mean_IU=float(miou),
               IU=torch.from_numpy(iu), pngs=pngs)
    print("mean IU", float(miou), "classes present", int((iu > 0).sum()))
    buf = io.BytesIO()
    torch.save(out, buf)
    with open(OUT, "wb") as f:
        f.write(gzip.compress(buf.getvalue(), 9, mtime=0))
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KB")


if __name__ == "__main__":
    main()
