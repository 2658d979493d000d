"""CPU: multi-scale / flip evaluation and test-split prediction maps -- the zoom rule the CUDA kernel implements against
scipy.ndimage.zoom bit for bit, the restatement in oracle/make_golden_eval.py against the fixture made by the UNMODIFIED reference,
the palette and Cityscapes id tables, and the public surface (imports, header, the ValueErrors of evaluate_main)."""
import gzip
import io
import os

import numpy as np
import pytest
import scipy.ndimage as nd
import torch

from oracle import make_golden_eval as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gold():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "eval_ms.pt.gz"), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def test_zoom_rule_is_bit_exact_with_scipy():
    rng = np.random.default_rng(0)
    cases = [(100, 161, s) for s in (0.5, 0.75, 1.0, 1.25, 1.5, 1.75)] + [(64, 96, 1.75), (1, 7, 2.0), (5, 1, 0.5)]
    for _ in range(60):
        cases.append((int(rng.integers(1, 200)), int(rng.integers(1, 200)), float(rng.choice([0.5, 0.75, 1.25, 1.5, 1.75, 0.3, 2.2]))))
    for H, W, s in cases:
        img = (rng.normal(0, 60, (1, 3, H, W))).astype(np.float32)
        ref = nd.zoom(img, (1.0, 1.0, s, s), order=1, prefilter=False)
        assert np.array_equal(G.zoom_rule(img, s), ref), (H, W, s)


def test_zoom_rule_zero_line_at_1024x2048():
    """767 * (1023 / 767) = 1023.0000000000001 > 1023: scipy's 'constant' mode returns row 767 as 0 at scale 0.75."""
    img = np.random.default_rng(1).normal(0, 60, (1, 3, 1024, 2048)).astype(np.float32)
    z = G.zoom_rule(img, 0.75)
    assert z.shape == (1, 3, 768, 1536)
    assert (z[:, :, 767] == 0).all() and (z[:, :, 766] != 0).any()
    assert np.array_equal(z, nd.zoom(img, (1.0, 1.0, 0.75, 0.75), order=1, prefilter=False))


def test_zoom_shape_is_scipys():
    from structure_knowledge_distillation_b200.networks.evaluate import zoom_shape
    for H, W, s in ((1024, 2048, 0.75), (100, 161, 1.75), (101, 33, 0.5), (7, 9, 1.25)):
        assert zoom_shape(H, W, s) == nd.zoom(np.zeros((1, 1, H, W), np.float32), (1, 1, s, s), order=1).shape[2:]


@pytest.mark.parametrize("key", ["100x161_flip0", "100x161_flip1", "64x96_flip0", "64x96_flip1"])
def test_restatement_matches_reference_golden(key):
    g = _gold()
    c = g["multiscale"][key]
    H, W = c["H"], c["W"]
    net = G.ToyNet().eval()
    got = G.predict_multiscale_rule(net, G.synth_image(H, W, c["image_seed"]), (H, W), g["scales"], c["flip"])
    ref = c["scores"].double().numpy()
    mine = got.reshape(H * W, -1)[c["positions"].numpy()]
    assert np.abs(mine - ref).max() <= 1e-6 * np.abs(ref).max()
    diff = np.argmax(got, 2) != c["argmax"].numpy()
    assert not (diff & (c["margin"].numpy() >= g["tie"])).any()


def test_golden_covers_the_zero_lines_and_near_ties():
    g = _gold()
    assert g["scales"] == (0.75, 1.0, 1.25, 1.75)
    assert set(g["multiscale"]) == {"100x161_flip0", "100x161_flip1", "64x96_flip0", "64x96_flip1"}
    assert sorted(g["test"]["pngs"]) == sorted(n for n, *_ in G.TEST_IMAGES)
    for name, p in g["test"]["pngs"].items():
        assert p["mode"] == "P" and tuple(p["pixels"].shape) == (1024, 2048)
        assert len(p["near_ties"]) < 1024 * 2048 // 1000                # near ties stay rare: the check has teeth
    assert [tuple(d["image"].shape) for d in g["dataset"]] == [(3, 64, 96), (3, 70, 100), (3, 64, 120)]
    assert os.path.getsize(os.path.join(ROOT, "tests", "golden", "eval_ms.pt.gz")) < 1 << 20


def test_palette_matches_the_reference_pngs():
    from structure_knowledge_distillation_b200.networks.evaluate import get_palette
    pal = get_palette(256)
    assert len(pal) == 768 and pal[:12] == [0, 0, 0, 128, 0, 0, 0, 128, 0, 128, 128, 0]
    g = _gold()
    for p in list(g["val"]["pngs"].values()) + list(g["test"]["pngs"].values()):
        assert p["palette"] == pal


def test_id_tables_come_from_one_source():
    """forward: the table the training loader applies (reference datasets.py:146-151); reverse: id2trainId(..., reverse=True) of
    evaluate.py:30-38 replayed on every uint8 value, with numpy 1's wrap of the table's -1 to 255."""
    from oracle.dataset_port import ID_TO_TRAINID, trainid_lut
    from structure_knowledge_distillation_b200.dataset import cityscapes_id_tables
    to_train, to_label = cityscapes_id_tables()
    assert np.array_equal(to_train, trainid_lut())
    lab = np.arange(256, dtype=np.int64)
    rev = lab.copy()
    for v, k in ID_TO_TRAINID.items():
        rev[lab == k] = v
    assert np.array_equal(to_label, (rev % 256).astype(np.uint8))
    assert np.array_equal(to_train[to_label[:19]], np.arange(19))
    # the test PNGs of the fixture hold label ids only
    used = set()
    for p in _gold()["test"]["pngs"].values():
        used |= set(np.unique(p["pixels"].numpy()).tolist())
    assert used <= set(to_label[:19].tolist()) and len(used) > 3


def test_test_set_returns_raw_files(tmp_path):
    import cv2
    from structure_knowledge_distillation_b200.dataset import CSDataTestSet
    g = _gold()["dataset"]
    for j, d in enumerate(g):
        assert cv2.imwrite(str(tmp_path / ("s%d.png" % j)), d["raw"].numpy())
    (tmp_path / "t.lst").write_text("".join("s%d.png\n" % j for j in range(len(g))))
    ds = CSDataTestSet(str(tmp_path), str(tmp_path / "t.lst"), crop_size=G.DATASET_CROP)
    assert len(ds) == len(g) and ds.mean == (104.00698793, 116.66876762, 122.67891434)
    for j, d in enumerate(g):
        image, size, name = ds[j]
        assert image.dtype == torch.uint8 and torch.equal(image, d["raw"])
        assert tuple(size) == d["size"] and name == d["name"]


def test_evaluate_main_refuses_what_the_reference_does_not_define():
    from structure_knowledge_distillation_b200.networks import evaluate as E
    net = torch.nn.Conv2d(3, 19, 1)
    for bad in ((), (0.5, 0.0), (-1.0,)):
        with pytest.raises(ValueError, match="scales"):
            E.evaluate_main(net, [], 0, "64,96", 19, whole=True, scales=bad)
    with pytest.raises(ValueError, match="whole=True"):
        E.evaluate_main(net, [], 0, "64,96", 19, whole=False, scales=(0.5, 1.0))
    with pytest.raises(ValueError, match="whole=True"):
        E.evaluate_main(net, [], 0, "64,96", 19, whole=False, flip=True)
    with pytest.raises(ValueError, match="19"):
        E.evaluate_main(net, [], 0, "64,96", 21, whole=True, type="test", png_dir="unused")
    with pytest.raises(ValueError, match="scales"):
        E.predict_multiscale(net, torch.zeros(1, 3, 8, 8), (8, 8), [], False, torch.zeros(8, 8, 19))


def test_public_surface_and_header():
    import inspect
    from structure_knowledge_distillation_b200 import _cabi, dataset
    from structure_knowledge_distillation_b200.networks import evaluate as E
    assert inspect.signature(E.predict_multiscale).parameters.keys() == {"model", "image", "tile_size", "scales", "flip", "full"}
    p = inspect.signature(E.evaluate_main).parameters
    assert p["scales"].default == (1.0,) and p["flip"].default is False and p["png_dir"].default is None and p["save_dir"].default is None
    assert dataset.CSDataTestSet is dataset.datasets.CSDataTestSet
    sig = _cabi.parse_header()
    new = {"skd_eval_zoom_image": 8, "skd_eval_upsample_accumulate_ms": 16, "skd_eval_argmax_confusion_lut": 15,
           "skd_cityscapes_id_tables": 2, "skd_cs_test_preprocess": 8}
    for n, k in new.items():
        assert n in sig and len(sig[n][1]) == k, n
    # the existing entries keep their signatures
    assert len(sig["skd_eval_upsample_accumulate"][1]) == 15 and len(sig["skd_eval_argmax_confusion"][1]) == 12
    if os.path.exists(_cabi.LIB_PATH):
        import ctypes
        dll = ctypes.CDLL(_cabi.LIB_PATH)
        assert all(hasattr(dll, n) for n in new)
