"""GPU: multi-scale / flip evaluation and test-split prediction maps (csrc/eval.cu) against scipy and the fixture made by the
UNMODIFIED reference (oracle/make_golden_eval.py).  The toy network runs with TF32 off, so its scores are fp32-grade."""
import gzip
import io
import os

import numpy as np
import pytest
import scipy.ndimage as nd
import torch

from oracle import make_golden_eval as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    with gzip.open(os.path.join(ROOT, "tests", "golden", "eval_ms.pt.gz"), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _toy():
    return G.ToyNet().cuda().eval()


def _pixels_agree(got, ref, near_ties):
    """equal except at the reference's near-tie pixels (top-2 margin < 1e-4), where fp32 scores may pick the other class"""
    diff = np.flatnonzero(got.reshape(-1) != ref.reshape(-1))
    return np.isin(diff, near_ties).all(), diff


@pytest.mark.parametrize("H,W", [(1024, 2048), (100, 161), (64, 96), (37, 5), (5, 53)])
def test_zoom_kernel_is_scipy_bit_for_bit(H, W):
    from structure_knowledge_distillation_b200.networks.evaluate import zoom_image
    img = np.random.default_rng(H * 7 + W).normal(0, 60, (1, 3, H, W)).astype(np.float32)
    dev = torch.from_numpy(img).cuda()
    for s in (0.5, 0.75, 1.25, 1.75):
        ref = nd.zoom(img, (1.0, 1.0, s, s), order=1, prefilter=False)[0].transpose(1, 2, 0)
        out = zoom_image(dev, s, flip=True)
        assert out.shape[:2] == (2, 4) and out.shape[2:] == ref.shape[:2]
        nhwc = out.permute(0, 2, 3, 1).cpu().numpy()
        assert np.array_equal(nhwc[0, ..., :3], ref), (H, W, s)
        assert np.array_equal(nhwc[1, ..., :3], ref[:, ::-1]), (H, W, s)
        assert (nhwc[..., 3] == 0).all()
        if (H, W, s) == (1024, 2048, 0.75):
            assert (nhwc[:, 767] == 0).all() and (nhwc[0, 766, :, :3] != 0).any()


def test_test_preprocess_is_bit_identical_to_the_fixture(gold):
    from structure_knowledge_distillation_b200.dataset import CSDataTestSet, DeviceTestPreprocess
    pre = DeviceTestPreprocess(G.DATASET_CROP, CSDataTestSet.MEAN)
    for d in gold["dataset"]:
        got = pre([d["raw"]])
        assert got.shape[0] == 1 and torch.equal(got[0].cpu(), d["image"]), d["size"]


@pytest.mark.parametrize("key", ["100x161_flip0", "100x161_flip1", "64x96_flip0", "64x96_flip1"])
def test_multiscale_scores_match_the_reference(gold, no_tf32, key):
    from structure_knowledge_distillation_b200._cabi import lib
    from structure_knowledge_distillation_b200.networks.evaluate import predict_multiscale
    c = gold["multiscale"][key]
    H, W = c["H"], c["W"]
    image = torch.from_numpy(G.synth_image(H, W, c["image_seed"])).cuda()
    full = torch.zeros(H, W, 19, device="cuda")
    predict_multiscale(_toy(), image, (H, W), gold["scales"], c["flip"], full)
    ref = c["scores"].double().numpy()
    got = full.reshape(H * W, 19)[c["positions"].cuda()].double().cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max(), np.abs(got - ref).max()
    pred = torch.empty(H, W, dtype=torch.uint8, device="cuda")
    conf = torch.zeros(19, 19, dtype=torch.int64, device="cuda")
    lib().skd_eval_argmax_confusion_lut(H, W, 19, full.data_ptr(), None, 0, 0, 0, 255, conf.data_ptr(), pred.data_ptr(), H, W, None,
                                        torch.cuda.current_stream().cuda_stream)
    ties = np.flatnonzero(c["margin"].numpy() < gold["tie"])
    ok, diff = _pixels_agree(pred.cpu().numpy(), c["argmax"].numpy(), ties)
    assert ok, diff[:20]
    # a second run is bit-identical
    full2 = torch.zeros_like(full)
    predict_multiscale(_toy(), image, (H, W), gold["scales"], c["flip"], full2)
    assert torch.equal(full, full2)


def _check_pngs(ref_pngs, d):
    from PIL import Image
    assert sorted(os.path.splitext(f)[0] for f in os.listdir(d)) == sorted(ref_pngs)
    for name, r in ref_pngs.items():
        im = Image.open(os.path.join(d, name + ".png"))
        assert im.mode == r["mode"] == "P" and list(im.getpalette()) == r["palette"]
        ok, diff = _pixels_agree(np.array(im), r["pixels"].numpy(), r["near_ties"].numpy())
        assert ok, (name, diff[:20])


def test_val_pngs_match_the_reference(gold, no_tf32, tmp_path):
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    miou, iu = evaluate_main(_toy(), G.val_batches(), 0, "64,96", 19, whole=False, png_dir=str(tmp_path))
    _check_pngs(gold["val"]["pngs"], tmp_path)
    assert abs(miou - gold["val"]["mean_IU"]) < 1e-3


def test_test_split_pngs_match_the_reference(gold, no_tf32, tmp_path):
    """test.py with the documented changes: CSDataTestSet + CSDataLoader + evaluate_main(whole=True, type='test', png_dir)."""
    import cv2
    from structure_knowledge_distillation_b200.dataset import CSDataLoader, CSDataTestSet, cityscapes_id_tables
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    data_dir = tmp_path / "cityscapes"
    lst = G.write_test_split(str(data_dir))
    ds = CSDataTestSet(str(data_dir), lst, crop_size=G.TEST_CROP)
    for k in range(len(ds)):
        name = ds.files[k]["name"]
        assert int(cv2.imread(ds.files[k]["img"]).astype(np.int64).sum()) == gold["test"]["pngs"][name]["raw_checksum"]
    loader = CSDataLoader(ds, batch_size=1, shuffle=False, pin_memory=True)
    images, size, names = next(iter(loader))
    assert images.is_cuda and tuple(images.shape) == (1, 3, 1024, 2048) and isinstance(names, list)
    out = tmp_path / "outputs"
    evaluate_main(_toy(), loader, '0', '512,512', 19, True, type='test', png_dir=str(out))
    _check_pngs(gold["test"]["pngs"], out)
    labels = set(cityscapes_id_tables()[1][:19].tolist())
    from PIL import Image
    for f in os.listdir(out):
        assert set(np.unique(np.array(Image.open(out / f))).tolist()) <= labels


def test_default_arguments_run_the_existing_path():
    """evaluate_main(scales=(1.0,), flip=False) gives the confusion matrix of predict_whole / predict_sliding +
    skd_eval_argmax_confusion driven directly, bit for bit, and launches no zoom kernel."""
    from structure_knowledge_distillation_b200._cabi import lib
    from structure_knowledge_distillation_b200.networks import evaluate as E
    net = _toy()
    g = torch.Generator().manual_seed(9)
    for whole, sizes, tile in ((True, ((1024, 2048),), (1024, 2048)), (False, ((100, 161), (130, 97)), (64, 96))):
        batches = []
        for i, (H, W) in enumerate(sizes):
            label = torch.randint(0, 19, (1, H, W), generator=g)
            label[torch.rand(1, H, W, generator=g) < 0.1] = 255
            batches.append((torch.from_numpy(G.synth_image(H, W, 50 + i)), label, [np.array([H - i, W - 2 * i, 3])], ["d%d" % i]))
        calls = []
        orig = E.zoom_image
        E.zoom_image = lambda *a, **k: calls.append(a) or orig(*a, **k)
        try:
            miou, iu = E.evaluate_main(net, batches, 0, "64,96", 19, whole=whole)
        finally:
            E.zoom_image = orig
        assert not calls
        conf = torch.zeros(19, 19, dtype=torch.int64, device="cuda")
        for image, label, size, _ in batches:
            image = image.cuda()
            H, W = image.shape[2:]
            full = torch.zeros(H, W, 19, device="cuda")
            (E.predict_whole if whole else E.predict_sliding)(net, image, tile, full)
            gt = label[0].cuda().long().contiguous()
            lib().skd_eval_argmax_confusion(H, W, 19, full.data_ptr(), gt.data_ptr(), W, int(min(size[0][0], H)), int(min(size[0][1], W)), 255,
                                            conf.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
        cm = conf.cpu().numpy().astype(np.float64)
        ref_iu = np.diag(cm) / np.maximum(1.0, cm.sum(1) + cm.sum(0) - np.diag(cm))
        assert np.array_equal(iu, ref_iu) and miou == ref_iu.mean()


def test_argmax_lut_counts_the_valid_region_and_maps_the_whole_image():
    from structure_knowledge_distillation_b200._cabi import lib
    from structure_knowledge_distillation_b200.dataset import cityscapes_id_tables
    H, W, vh, vw = 37, 53, 30, 41
    g = torch.Generator().manual_seed(4)
    full = torch.randn(H, W, 19, generator=g).cuda()
    gt = torch.randint(0, 19, (H, W), generator=g)
    gt[torch.rand(H, W, generator=g) < 0.2] = 255
    gt = gt.cuda()
    lut = torch.from_numpy(cityscapes_id_tables()[1]).cuda()
    st = torch.cuda.current_stream().cuda_stream
    conf_a = torch.zeros(19, 19, dtype=torch.int64, device="cuda")
    conf_b = torch.zeros_like(conf_a)
    pred_a = torch.empty(H, W, dtype=torch.uint8, device="cuda")
    pred_b = torch.empty_like(pred_a)
    lib().skd_eval_argmax_confusion(H, W, 19, full.data_ptr(), gt.data_ptr(), W, vh, vw, 255, conf_a.data_ptr(), pred_a.data_ptr(), st)
    lib().skd_eval_argmax_confusion_lut(H, W, 19, full.data_ptr(), gt.data_ptr(), W, vh, vw, 255, conf_b.data_ptr(), pred_b.data_ptr(), H, W,
                                        lut.data_ptr(), st)
    am = full.argmax(2)
    assert torch.equal(conf_a, conf_b)
    assert torch.equal(pred_b, lut[am])
    assert torch.equal(pred_a[:vh, :vw], am[:vh, :vw].to(torch.uint8))


def test_png_writer_errors_reach_the_caller(tmp_path):
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    H, W = 64, 96
    batches = [(torch.from_numpy(G.synth_image(H, W, 1)), torch.zeros(1, H, W, dtype=torch.long), [np.array([H, W, 3])], ["no_such_dir/x"])]
    with pytest.raises(FileNotFoundError):
        evaluate_main(_toy(), batches, 0, "64,96", 19, whole=False, png_dir=str(tmp_path))


def test_student_flip_batch_matches_two_single_forwards():
    """The real student at 1024x2048: the batch-2 (image, mirror) forward against two batch-1 forwards.  Eval-mode BN is per
    image, so only the convolutions' tiling could differ; stated tolerance 1e-6 relative (L2).  Two multi-scale runs are
    bit-identical."""
    from structure_knowledge_distillation_b200.networks.evaluate import predict_multiscale, zoom_image
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Res_pspnet
    torch.manual_seed(0)
    net = Res_pspnet(BasicBlock, [2, 2, 2, 2], 19).cuda().eval()
    image = torch.from_numpy(G.synth_image(1024, 2048, 5)).cuda()
    x = zoom_image(image, 1.0, flip=True)
    with torch.no_grad():
        both = net(x)[0].float()
        one = torch.cat([net(x[:1].contiguous(memory_format=torch.channels_last))[0].float(),
                         net(x[1:].contiguous(memory_format=torch.channels_last))[0].float()])
    rel = float((both - one).norm() / one.norm())
    assert rel <= 1e-6, rel
    fulls = []
    for _ in range(2):
        full = torch.zeros(1024, 2048, 19, device="cuda")
        predict_multiscale(net, image, (1024, 2048), (0.75, 1.0, 1.25), True, full)
        fulls.append(full)
    assert torch.equal(fulls[0], fulls[1])
    assert torch.isfinite(fulls[0]).all()
