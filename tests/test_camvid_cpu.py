"""CamVid without a GPU: the SegNet label table, list parsing, the ENet class-frequency weights on synthetic label PNGs, and every
ValueError of the class-weighted task loss (criteria, NetModel, SegModel), raised before any device work."""
import argparse

import numpy as np
import pytest
import torch


def test_camvid_label_table():
    from structure_knowledge_distillation_b200.dataset import CAMVID_CLASSES, camvid_label_table
    assert CAMVID_CLASSES == ("Sky", "Building", "Pole", "Road", "Pavement", "Tree", "SignSymbol", "Fence", "Car", "Pedestrian",
                              "Bicyclist")
    t = camvid_label_table()
    assert t.dtype == np.uint8 and t.shape == (256,)
    assert np.array_equal(t[:11], np.arange(11)) and (t[11:] == 255).all()
    t7 = camvid_label_table(ignore_label=200)
    assert np.array_equal(t7[:11], np.arange(11)) and (t7[11:] == 200).all()


def _write_camvid(tmp_path, labels, cv2):
    (tmp_path / "train").mkdir(); (tmp_path / "trainannot").mkdir()
    lines = []
    for i, lab in enumerate(labels):
        img = np.zeros(lab.shape + (3,), np.uint8)
        cv2.imwrite(str(tmp_path / "train" / ("f%d.png" % i)), img)
        cv2.imwrite(str(tmp_path / "trainannot" / ("f%d.png" % i)), lab)
        lines.append("train/f%d.png trainannot/f%d.png\n" % (i, i))
    (tmp_path / "train.txt").write_text("".join(lines))
    return str(tmp_path), str(tmp_path / "train.txt")


def test_camvid_list_parsing(tmp_path):
    from structure_knowledge_distillation_b200.dataset import CamVidDataSet, CSDataSet
    (tmp_path / "train.txt").write_text("train/0001TP_006690.png trainannot/0001TP_006690.png\n"
                                        "val/Seq05VD_f00000.png  valannot/Seq05VD_f00000.png\n")
    ds = CamVidDataSet(str(tmp_path), str(tmp_path / "train.txt"))
    assert isinstance(ds, CSDataSet) and len(ds) == 2
    assert (ds.crop_h, ds.crop_w) == (360, 480) and ds.mean == (128, 128, 128) and ds.scale and ds.is_mirror and ds.ignore_label == 255
    assert ds.files[0] == {"img": str(tmp_path / "train/0001TP_006690.png"), "label": str(tmp_path / "trainannot/0001TP_006690.png"),
                           "name": "0001TP_006690"}
    assert ds.files[1]["name"] == "Seq05VD_f00000"
    assert len(CamVidDataSet(str(tmp_path), str(tmp_path / "train.txt"), max_iters=5)) == 6
    assert (CamVidDataSet(str(tmp_path), str(tmp_path / "train.txt"), ignore_label=11).label_table[11:] == 11).all()


def test_camvid_getitem_draws_like_cityscapes(tmp_path):
    """Same raw files and same random draws (CS_SCALES) as CSDataSet."""
    cv2 = pytest.importorskip("cv2")
    import random
    from structure_knowledge_distillation_b200.dataset import CamVidDataSet, CSDataSet
    rng = np.random.default_rng(0)
    root, lst = _write_camvid(tmp_path, [rng.integers(0, 256, (37, 53), dtype=np.uint8)], cv2)
    outs = []
    for cls in (CamVidDataSet, CSDataSet):
        random.seed(4); np.random.seed(4)
        outs.append(cls(root, lst, crop_size=(20, 30))[0])
    for a, b in zip(outs[0][:4], outs[1][:4]):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    assert outs[0][4] == outs[1][4] == "f0"


def test_class_frequency_weights_formula(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset import CamVidDataSet, VOCDataSet, class_frequency_weights
    rng = np.random.default_rng(1)
    labels = [rng.integers(0, 256, (24, 31), dtype=np.uint8), rng.choice(np.array([0, 3, 3, 3, 11, 10, 200], np.uint8), (17, 40))]
    root, lst = _write_camvid(tmp_path, labels, cv2)
    ds = CamVidDataSet(root, lst, max_iters=7)                        # a repeated list still reads each file once
    counts = np.zeros(11)
    for lab in labels:
        for k in range(11):
            counts[k] += (lab == k).sum()
    p = counts / counts.sum()
    for c in (1.02, 1.1):
        w = class_frequency_weights(ds, 11, c)
        assert w.dtype == np.float32 and w.shape == (11,)
        assert np.array_equal(w, (1.0 / np.log(c + p)).astype(np.float32)), (w, 1.0 / np.log(c + p))
    assert w[3] == w.min()                                             # the most frequent class gets the smallest weight
    # any dataset: a VOC loader has no table, so labels 0..20 count as they are
    (tmp_path / "JPEGImages").mkdir(); (tmp_path / "SegmentationClassAug").mkdir()
    vlab = rng.integers(0, 22, (20, 20), dtype=np.uint8); vlab[:3] = 255
    cv2.imwrite(str(tmp_path / "SegmentationClassAug" / "a.png"), vlab)
    (tmp_path / "voc.txt").write_text("a\n")
    vc = np.array([(vlab == k).sum() for k in range(21)], np.float64)
    wv = class_frequency_weights(VOCDataSet(str(tmp_path), str(tmp_path / "voc.txt")), 21)
    assert np.array_equal(wv, (1.0 / np.log(1.02 + vc / vc.sum())).astype(np.float32))


def test_class_frequency_weights_errors(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset import CamVidDataSet, class_frequency_weights
    root, lst = _write_camvid(tmp_path, [np.full((8, 8), 11, np.uint8)], cv2)
    with pytest.raises(ValueError, match="no labelled pixel"):
        class_frequency_weights(CamVidDataSet(root, lst), 11)
    (tmp_path / "bad.txt").write_text("train/f0.png trainannot/missing.png\n")
    with pytest.raises(IOError, match="missing.png"):
        class_frequency_weights(CamVidDataSet(root, str(tmp_path / "bad.txt")), 11)


W11 = [0.5] * 11


@pytest.mark.parametrize("weight,msg", [
    ([1.0] * 10, "10 entries for 11 classes"),
    ([1.0] * 12, "12 entries for 11 classes"),
    ([1.0] * 10 + [-0.5], "non-negative"),
    ([1.0] * 10 + [float("nan")], "finite"),
    ([1.0] * 10 + [float("inf")], "finite"),
    ([0.0] * 11, "all zero"),
    (torch.zeros(11), "all zero"),
    ([[1.0] * 11], "1-D"),
    (["a"] * 11, "floats"),
])
@pytest.mark.parametrize("model", ["NetModel", "SegModel"])
def test_model_class_weight_validation(model, weight, msg):
    """args.class_weights is checked next to classes_num, before any device work."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    args = argparse.Namespace(classes_num=11, class_weights=weight, device=torch.device("cuda"))
    with pytest.raises(ValueError, match=msg):
        (NetModel if model == "NetModel" else SegModel)(args)


@pytest.mark.parametrize("model", ["NetModel", "SegModel"])
def test_class_weights_with_ohem_raise(model):
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    args = argparse.Namespace(classes_num=11, class_weights=W11, ohem=True, device=torch.device("cuda"))
    with pytest.raises(ValueError, match="ohem"):
        (NetModel if model == "NetModel" else SegModel)(args)


def test_criterion_class_weight_validation():
    from structure_knowledge_distillation_b200.utils.criterion import CriterionCrossEntropy, CriterionDSN, check_class_weights
    for crit in (CriterionDSN, CriterionCrossEntropy):
        assert crit().weight is None
        for bad in ([1.0, -1.0], [float("nan")], [0.0, 0.0], []):
            with pytest.raises(ValueError):
                crit(weight=bad)
        c = crit(255, True, True, np.array([1, 2.5], np.float64))       # the new keyword comes last
        assert c.weight.dtype == torch.float32 and c.weight.tolist() == [1.0, 2.5] and c.weight.device.type == "cpu"
    w = check_class_weights(torch.tensor([0.0, 3.0], dtype=torch.float64), 2)
    assert w.dtype == torch.float32 and w.tolist() == [0.0, 3.0]
    assert check_class_weights(None, 19) is None
