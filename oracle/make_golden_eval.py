"""TEST INFRASTRUCTURE -- generates tests/golden/eval_ms.pt.gz by running the UNMODIFIED reference evaluation on CPU.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_eval        (needs cv2 and PIL)

Imported as shipped: networks/evaluate.py (predict_multiscale, evaluate_main) and dataset/datasets.py (CSDataTestSet).  Made to run
on CPU under numpy 2 at call time only:
  * `.cuda()` of tensors and modules is the identity (evaluate.py:109,166);
  * `np.int` is `int` while evaluate_main runs (evaluate.py:194, val path);
  * id2trainId(..., reverse=True) (evaluate.py:30-38,188) stores the table's -1 into a uint8 map; numpy 1 wrapped it to 255,
    numpy 2 raises OverflowError -- the shim runs the unmodified function on an int64 copy and wraps the result back to uint8.
The network is `ToyNet`, fixed-weight class scores at 1/8 resolution from plain torch ops (the evaluation path is what is under
test).  Recorded, with the restatement below pinned against the reference on the spot:
  * predict_multiscale at scales (0.75, 1.0, 1.25, 1.75), with and without flip, on 100x161 (scipy's zero row 74 at 0.75 and
    column 281 at 1.75) and 64x96: arg-max, top-2 margin, and the scores at a seeded sample of pixels;
  * evaluate_main(type='val') (sliding tiles) and the test.py flow -- CSDataTestSet + DataLoader + evaluate_main(whole=True,
    type='test') on 1024x2048 images -- PNGs read back as pixel arrays and palette, plus the pixels whose top-2 margin is < 1e-4;
  * CSDataTestSet.__getitem__ for images smaller than, larger than and across the crop.
"""
import contextlib
import gzip
import importlib
import io
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

from .refshim import REFERENCE_ROOT

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "eval_ms.pt.gz")
MS_SCALES = (0.75, 1.0, 1.25, 1.75)
MS_SIZES = ((100, 161), (64, 96))
SAMPLES = 1000
TIE = 1e-4
VAL_SIZES = ((100, 161), (130, 97))          # sliding tiles of 64x96
TEST_IMAGES = (("frankfurt_000000_000294_leftImg8bit", 1024, 2048, 11), ("lindau_000000_000019_leftImg8bit", 1000, 2000, 12))
TEST_CROP = (1024, 2048)                     # test.py:9
DATASET_CASES = ((50, 80), (70, 100), (60, 120))
DATASET_CROP = (64, 96)


class ToyNet(torch.nn.Module):
    """19-class scores at 1/8 resolution: a 1x1 convolution of the 8x8 average-pooled colour channels.  Takes the 3-channel image
    or the 4-channel (zero 4th channel) network input."""

    def __init__(self, classes=19):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.w = torch.nn.Parameter(torch.randn(classes, 3, 1, 1, generator=g) * 0.05)
        self.b = torch.nn.Parameter(torch.randn(classes, generator=g) * 0.5)

    def forward(self, x):
        return [F.conv2d(F.avg_pool2d(x[:, :3], 8, 8, ceil_mode=True), self.w, self.b)]


def synth_image(H, W, seed):
    """float32 (1, 3, H, W), mean-subtracted-looking values: smooth colour fields plus noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    base = np.stack([60 * np.sin(xx / 17.0 + c) + 50 * np.cos(yy / 11.0 - 2 * c) for c in range(3)])
    return (base + rng.normal(0, 25, (3, H, W)))[None].astype(np.float32)


def raw_image(H, W, seed):
    """uint8 H x W x 3 BGR file content: coarse random blocks, blurred by resampling, plus noise."""
    rng = np.random.default_rng(seed)
    coarse = rng.integers(0, 256, (H // 64 + 2, W // 64 + 2, 3)).astype(np.float64)
    t = torch.from_numpy(coarse).permute(2, 0, 1)[None]
    smooth = F.interpolate(t, size=(H, W), mode="bilinear", align_corners=True)[0].permute(1, 2, 0).numpy()
    return np.clip(smooth + rng.normal(0, 12, (H, W, 3)), 0, 255).astype(np.uint8)


# ----------------------------------------------------------------------------------------------------------- restatement
def zoom_rule(image, scale):
    """scipy.ndimage.zoom(image, (1, 1, s, s), order=1, prefilter=False) of a float32 (1, C, H, W) array, written out as the zoom
    kernel computes it (csrc/common.cuh zoom_axis / zoom_lerp): coordinate o * (in-1)/(out-1) in double, 0 past the last row or
    column (mode 'constant'), the four neighbours times their weights summed in scipy's order, rounded to float32."""
    _, _, H, W = image.shape
    oh, ow = int(round(H * scale)), int(round(W * scale))

    def axis(n_in, n_out):
        r = (n_in - 1) / (n_out - 1) if n_out > 1 else 1.0
        c = np.arange(n_out, dtype=np.float64) * r
        i0 = np.floor(c).astype(np.int64)
        i1 = np.minimum(i0 + 1, n_in - 1)
        i0 = np.minimum(i0, n_in - 1)
        t = c - i0
        return i0, i1, t, 1.0 - t, c > n_in - 1

    y0, y1, ty, wy, oy = axis(H, oh)
    x0, x1, tx, wx, ox = axis(W, ow)
    P = image.astype(np.float64)
    Y0, Y1, TY, WY = y0[:, None], y1[:, None], ty[:, None], wy[:, None]
    v = P[..., Y0, x0] * WY * wx
    v = v + P[..., Y0, x1] * WY * tx
    v = v + P[..., Y1, x0] * TY * wx
    v = v + P[..., Y1, x1] * TY * tx
    v[..., oy, :] = 0
    v[..., :, ox] = 0
    return v.astype(np.float32)


@torch.no_grad()
def predict_multiscale_rule(net, image, tile, scales, flip):
    """predict_multiscale (evaluate.py:115-134) with the zoom restated: -> (H, W, C) float64."""
    full = None
    for s in scales:
        z = torch.from_numpy(zoom_rule(image, s))
        up = lambda x: F.interpolate(net(x)[0], size=tile, mode="bilinear", align_corners=True)[0].permute(1, 2, 0).numpy()
        p = up(z)
        if flip:
            p = 0.5 * (p + up(z.flip(3))[:, ::-1, :])
        full = p.astype(np.float64) if full is None else full + p
    return full / len(scales)


def top2_margin(scores):
    s = np.sort(scores, axis=-1)
    return (s[..., -1] - s[..., -2]).astype(np.float32)


def sample_positions(H, W, seed):
    return np.random.default_rng(seed).choice(H * W, size=min(SAMPLES, H * W), replace=False)


# ----------------------------------------------------------------------------------------------------------- reference
def load_reference_eval():
    """-> (networks.evaluate, dataset.datasets) of the reference, imported as shipped."""
    from . import refshim
    refshim.load_reference()                                          # installs the `libs` / `tensorboardX` import shims
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k.split(".")[0] in ("networks", "dataset", "utils")}
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        ev = importlib.import_module("networks.evaluate")
        ds = importlib.import_module("dataset.datasets")
    finally:
        sys.path.remove(REFERENCE_ROOT)
        for k in list(sys.modules):
            if k.split(".")[0] in ("networks", "dataset", "utils"):
                del sys.modules[k]
        sys.modules.update(saved)
    return ev, ds


@contextlib.contextmanager
def cpu_numpy2_shims(ev):
    orig = (torch.Tensor.cuda, torch.nn.Module.cuda, ev.id2trainId, getattr(np, "int", None))
    orig_id = ev.id2trainId
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    ev.id2trainId = lambda label, table, reverse=False: orig_id(label.astype(np.int64), table, reverse).astype(np.uint8)
    np.int = int
    try:
        yield
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda, ev.id2trainId = orig[:3]
        del np.int


def read_pngs(d):
    from PIL import Image
    out = {}
    for f in sorted(os.listdir(d)):
        im = Image.open(os.path.join(d, f))
        out[os.path.splitext(f)[0]] = dict(mode=im.mode, pixels=torch.from_numpy(np.array(im)), palette=list(im.getpalette()))
    return out


def val_batches():
    g = torch.Generator().manual_seed(3)
    batches = []
    for i, (H, W) in enumerate(VAL_SIZES):
        image = torch.from_numpy(synth_image(H, W, 40 + i))
        label = torch.randint(0, 19, (1, H, W), generator=g)
        label[torch.rand(1, H, W, generator=g) < 0.1] = 255
        size = torch.tensor([[H, W, 3]])                              # evaluate.py:194-197 crops the label only
        batches.append((image, label, size, ["val%d" % i]))
    return batches


def write_test_split(root):
    """the raw test files and test.lst (one 'leftImg8bit/test/<city>/<name>.png' path per line) -> list path"""
    import cv2
    lines = []
    for name, H, W, seed in TEST_IMAGES:
        rel = os.path.join("leftImg8bit", "test", name.split("_")[0], name + ".png")
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        assert cv2.imwrite(os.path.join(root, rel), raw_image(H, W, seed))
        lines.append(rel)
    lst = os.path.join(root, "test.lst")
    with open(lst, "w") as f:
        f.write("\n".join(lines) + "\n")
    return lst


def main():
    import cv2
    from torch.utils import data
    ev, ds = load_reference_eval()
    torch.set_num_threads(os.cpu_count())
    net = ToyNet().eval()
    out = dict(scales=MS_SCALES, tie=TIE, multiscale={}, cv2=cv2.__version__)
    cwd = os.getcwd()
    with cpu_numpy2_shims(ev), torch.no_grad(), tempfile.TemporaryDirectory() as tmp:
        # predict_multiscale
        for i, (H, W) in enumerate(MS_SIZES):
            image = synth_image(H, W, 20 + i)
            for flip in (False, True):
                for s in MS_SCALES:                                       # the restated zoom is scipy's, bit for bit
                    import scipy.ndimage as nd
                    assert np.array_equal(zoom_rule(image, s), nd.zoom(image, (1.0, 1.0, s, s), order=1, prefilter=False)), (H, W, s)
                ref = ev.predict_multiscale(net, torch.from_numpy(image), (H, W), list(MS_SCALES), 19, flip, 1)
                mine = predict_multiscale_rule(net, image, (H, W), MS_SCALES, flip)
                assert np.abs(mine - ref).max() <= 1e-6 * np.abs(ref).max(), (H, W, flip)
                pos = sample_positions(H, W, 7 + i)
                out["multiscale"]["%dx%d_flip%d" % (H, W, flip)] = dict(
                    H=H, W=W, flip=flip, image_seed=20 + i, argmax=torch.from_numpy(np.argmax(ref, 2).astype(np.uint8)),
                    margin=torch.from_numpy(top2_margin(ref)), positions=torch.from_numpy(pos),
                    scores=torch.from_numpy(ref.reshape(H * W, -1)[pos].astype(np.float32)))
                print("multiscale", H, W, "flip", flip, "near ties", int((top2_margin(ref) < TIE).sum()))
        # evaluate_main(type='val'): sliding tiles, train-id PNGs in ./outputs
        os.chdir(os.path.join(tmp))
        try:
            os.makedirs("val"); os.chdir("val")
            miou, iu = ev.evaluate_main(net, val_batches(), "0", "64,96", 19, False, type="val")
            pngs = read_pngs("outputs")
            for image, _, _, name in val_batches():
                scores = ev.predict_sliding(net, image.numpy(), (64, 96), 19, False, 1)
                pngs[name[0]]["near_ties"] = torch.from_numpy(np.flatnonzero(top2_margin(scores) < TIE))
            out["val"] = dict(mean_IU=float(miou), IU=torch.from_numpy(iu), pngs=pngs)
            os.chdir(tmp)
            # test.py: CSDataTestSet + DataLoader + evaluate_main(whole=True, type='test'): label-id PNGs
            data_dir = os.path.join(tmp, "cityscapes")
            lst = write_test_split(data_dir)
            ts = ds.CSDataTestSet(data_dir, lst, crop_size=TEST_CROP)
            loader = data.DataLoader(ts, batch_size=1, shuffle=False, pin_memory=False)
            os.makedirs("test"); os.chdir("test")
            ev.evaluate_main(net, loader, "0", "512,512", 19, True, type="test")
            pngs = read_pngs("outputs")
            for k in range(len(ts)):
                image, size, name = ts[k]
                scores = ev.predict_multiscale(net, torch.from_numpy(image[None]), TEST_CROP, [1.0], 19, False, 1)
                pngs[name]["near_ties"] = torch.from_numpy(np.flatnonzero(top2_margin(scores) < TIE))
                pngs[name]["raw_checksum"] = int(cv2.imread(ts.files[k]["img"]).astype(np.int64).sum())
            out["test"] = dict(images=TEST_IMAGES, crop=TEST_CROP, pngs=pngs)
            # CSDataTestSet.__getitem__ on small images
            out["dataset"] = []
            small = os.path.join(tmp, "small")
            os.makedirs(small)
            for j, (H, W) in enumerate(DATASET_CASES):
                raw = raw_image(H, W, 30 + j)
                assert cv2.imwrite(os.path.join(small, "s%d.png" % j), raw)
                with open(os.path.join(small, "s.lst"), "w") as f:
                    f.write("s%d.png\n" % j)
                image, size, name = ds.CSDataTestSet(small, os.path.join(small, "s.lst"), crop_size=DATASET_CROP)[0]
                out["dataset"].append(dict(raw=torch.from_numpy(raw), crop=DATASET_CROP, image=torch.from_numpy(np.ascontiguousarray(image)),
                                           size=tuple(int(v) for v in size), name=name))
        finally:
            os.chdir(cwd)
    buf = io.BytesIO()
    torch.save(out, buf)
    with open(OUT, "wb") as f:
        f.write(gzip.compress(buf.getvalue(), 9, mtime=0))
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KB")


if __name__ == "__main__":
    main()
