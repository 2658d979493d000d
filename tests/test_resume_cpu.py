"""CPU: resuming a run.  The training-state file of StepModel (networks/step_model.py) -- its reference keys, the checks that refuse a file
of another model, the atomic write, the per-rank random streams over gloo -- on CPU stand-ins of NetModel / SegModel (same attributes,
no kernels), and CSDataLoader's resumable iteration (raw batches: names, files and augmentation draws, which the workers make on the
CPU) against an uninterrupted one."""
import os
import random
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _standin(seg=False, kind="resnet18", classes=19, seed=0):
    """A NetModel (or SegModel) as the training-state methods see it, on the CPU: network, FlatSGD solvers, discriminator (NetModel)."""
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.sagan_models import Discriminator
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    from structure_knowledge_distillation_b200.optim import FlatSGD
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(seed)
    m = object.__new__(SegModel if seg else NetModel)
    m.args = make_args(classes_num=classes, student=kind, seg_model=kind)
    m.device, m.world, m.best_mean_IU = torch.device("cpu"), 1, 0.0
    m.kind, m.kind_option = kind, "seg_model" if seg else "student"
    m._net = build_seg_network(kind, classes)
    m.G_solver = FlatSGD([p for p in m._net.parameters() if p.requires_grad], 0.01, momentum=0.9, weight_decay=5e-4)
    m.G_solver.flat_m.normal_()
    m.G_solver.steps = 7 + seed
    if not seg:
        m.D_model = Discriminator(1, classes, 2, 65, 64)
        m.D_solver = FlatSGD([p for p in m.D_model.parameters() if p.requires_grad], 4e-4, momentum=0.9, weight_decay=5e-4)
        m.D_solver.flat_m.normal_()
        with torch.no_grad():
            m.D_model.preprocess_additional.running_mean.normal_()
            m.D_model.l1[0].module.weight_u.normal_()
    return m


def _snapshot(m):
    """Everything load_training_state may touch."""
    parts = [m._net.state_dict(), m.G_solver.flat_m, m.G_solver.flat_p]
    if hasattr(m, "D_solver"):
        parts += [m.D_model.state_dict(), m.D_solver.flat_m, m.D_solver.flat_p]
    flat = []
    for p in parts:
        flat += [v.clone() for v in p.values()] if isinstance(p, dict) else [p.clone()]
    return flat, m.G_solver.steps, torch.get_rng_state(), random.getstate(), np.random.get_state()[1].copy()


def _same_snapshot(a, b):
    return (len(a[0]) == len(b[0]) and all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1] and torch.equal(a[2], b[2])
            and a[3] == b[3] and np.array_equal(a[4], b[4]))


def test_training_state_round_trip_restores_everything(tmp_path):
    src, dst = _standin(seed=0), _standin(seed=1)
    random.seed(3); np.random.seed(4); torch.manual_seed(5)
    want_rng = (torch.get_rng_state(), random.getstate(), np.random.get_state())
    src.save_training_state(str(tmp_path / "state.pth"), 1234, epoch=2, best_mean_IU=0.5, IU_array=np.arange(19) / 19)
    random.seed(30); np.random.seed(40); torch.manual_seed(50)
    assert dst.load_training_state(str(tmp_path / "state.pth")) == 1234
    assert _same_snapshot(_snapshot(dst), (_snapshot(src)[0], src.G_solver.steps) + _snapshot(dst)[2:])
    assert dst.D_solver.steps == src.D_solver.steps
    assert torch.equal(torch.get_rng_state(), want_rng[0]) and random.getstate() == want_rng[1]
    assert np.array_equal(np.random.get_state()[1], want_rng[2][1]) and np.random.get_state()[2] == want_rng[2][2]
    assert (dst.args.last_step, dst.args.start_epoch, dst.args.best_mean_IU, dst.best_mean_IU) == (1234, 2, 0.5, 0.5)


def test_reference_keys_load_through_load_S_model_and_load_seg_model(tmp_path):
    """Renamed to model_best.pth.tar, the file resumes the student (S_resume) and a SegModel network (resume) through the reference's
    loaders, counters included."""
    from structure_knowledge_distillation_b200.networks.step_model import build_seg_network
    from structure_knowledge_distillation_b200.utils import utils as U
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    for seg in (False, True):
        m = _standin(seg=seg)
        d = tmp_path / ("seg" if seg else "student")
        d.mkdir()
        m.save_training_state(str(d / "model_best.pth.tar"), 321, epoch=4, best_mean_IU=0.625, IU_array=np.linspace(0, 1, 19))
        net = build_seg_network("resnet18", 19)
        if seg:
            args = make_args(ckpt_path=str(d), resume=True)
            assert U.load_seg_model(args, net, False) == "resume"
        else:
            args = make_args(S_ckpt_path=str(d), S_resume=True)
            assert U.load_S_model(args, net, False) == "resume"
        assert (args.last_step, args.start_epoch, args.best_mean_IU) == (321, 4, 0.625)
        assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), m._net.state_dict().values()))
        ck = U._torch_load(str(d / "model_best.pth.tar"))
        assert np.array_equal(ck["IU_array"], np.linspace(0, 1, 19))


def _rewrite(path, **change):
    ck = torch.load(path, weights_only=False)
    for k, v in change.items():
        if "." in k:
            a, b = k.split(".")
            ck[a][b] = v
        else:
            ck[k] = v
    torch.save(ck, path)


@pytest.mark.parametrize("field,change", [
    ("version", dict(version=99)),
    ("kind", dict(kind=("student", "mobilenetv2"))),
    ("classes_num", dict(classes_num=21)),
    ("world_size", dict(world_size=2)),
    ("G_solver.numel", {"G_solver.numel": 12}),
    ("D_solver.numel", {"D_solver.numel": 12}),
    ("state_dict", {"state_dict.conv1.weight": torch.zeros(3)}),
    ("D_state_dict", {"D_state_dict.l1.0.module.weight_u": torch.zeros(3)}),
])
def test_mismatch_raises_and_leaves_model_untouched(tmp_path, field, change):
    path = str(tmp_path / "state.pth")
    _standin(seed=0).save_training_state(path, 10)
    if "state_dict." in next(iter(change)):
        key, v = next(iter(change.items()))
        sd, name = key.split(".", 1)
        ck = torch.load(path, weights_only=False)
        ck[sd][name] = v
        torch.save(ck, path)
    else:
        _rewrite(path, **change)
    dst = _standin(seed=1)
    before = _snapshot(dst)
    with pytest.raises(ValueError, match=field.split(".")[0]):
        dst.load_training_state(path)
    assert _same_snapshot(_snapshot(dst), before)
    assert dst.args.last_step == 0


def test_other_model_files_are_refused(tmp_path):
    """A SegModel file into NetModel (kind), 19 classes into a 21-class model, a loader position the file does not have."""
    path, path2 = str(tmp_path / "seg.pth"), str(tmp_path / "c19.pth")
    _standin(seg=True).save_training_state(path, 5)
    _standin().save_training_state(path2, 5)
    dst, c21 = _standin(seed=1), _standin(classes=21)

    class _Loader:
        def load_state_dict(self, sd):
            raise AssertionError("not reached")
    before, before21 = _snapshot(dst), _snapshot(c21)
    with pytest.raises(ValueError, match="kind"):
        dst.load_training_state(path)
    with pytest.raises(ValueError, match="classes_num"):
        c21.load_training_state(path2)
    with pytest.raises(ValueError, match="loader"):
        dst.load_training_state(path2, loader=_Loader())
    assert _same_snapshot(_snapshot(dst), before) and _same_snapshot(_snapshot(c21), before21)


def test_interrupted_write_leaves_previous_file(tmp_path, monkeypatch):
    path = str(tmp_path / "state.pth")
    m = _standin()
    m.save_training_state(path, 100)
    before = open(path, "rb").read()
    real_save = torch.save

    def dying_save(obj, f, *a, **k):
        f.write(b"partial")
        raise OSError("disk full")
    monkeypatch.setattr(torch, "save", dying_save)
    with pytest.raises(RuntimeError, match="disk full"):
        m.save_training_state(path, 200)
    monkeypatch.setattr(torch, "save", real_save)
    assert open(path, "rb").read() == before
    assert os.listdir(tmp_path) == ["state.pth"]                     # the temporary file is gone
    assert _standin(seed=1).load_training_state(path) == 100


_GLOO = textwrap.dedent('''
    import os, random, sys, numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    sys.path.insert(0, os.path.join(%r, "tests"))
    from test_resume_cpu import _standin, _snapshot, _same_snapshot
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    path = sys.argv[1]
    m = _standin(seed=0); m.world = world
    random.seed(10 + rank); np.random.seed(20 + rank); torch.manual_seed(30 + rank)
    mine = (torch.get_rng_state(), random.getstate(), np.random.get_state()[1].copy())
    m.save_training_state(path, 77)
    assert os.path.isfile(path)                                      # complete on every rank when the call returns
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    d = _standin(seed=1); d.world = world
    assert d.load_training_state(path) == 77
    assert torch.equal(torch.get_rng_state(), mine[0]) and random.getstate() == mine[1] and np.array_equal(np.random.get_state()[1], mine[2])
    assert all(torch.equal(a, b) for a, b in zip(_snapshot(d)[0], _snapshot(m)[0]))
    ck = torch.load(path, weights_only=False)
    assert ck["world_size"] == world and len(ck["ranks"]) == world
    assert not torch.equal(ck["ranks"][0]["torch"], ck["ranks"][1]["torch"])
    one = _standin(seed=2)
    try:
        one.load_training_state(path)                                # world size 1
        raise SystemExit("world_size mismatch not detected")
    except ValueError as e:
        assert "world_size" in str(e)
    dist.barrier(); dist.destroy_process_group()
    print("rank", rank, "ok")
''')


def test_per_rank_random_streams_gather_gloo_world2(tmp_path):
    """Two gloo ranks with different random streams: rank 0 writes one file holding both, each rank gets its own streams back, and a
    one-process model refuses the two-rank file."""
    script = tmp_path / "resume_ddp.py"
    script.write_text(_GLOO % (ROOT, ROOT))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29547", str(script), str(tmp_path / "state.pth")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("ok") == 2


# ---- CSDataLoader ----------------------------------------------------------------------------------------------------------------
SIZES = [(40, 60), (52, 71), (33, 47), (64, 96), (45, 45), (70, 38)]


def _write_dataset(root, style, n=11):
    """`n` image / label pairs of mixed sizes in the Cityscapes (list of 'image label' paths, PNG) or VOC (names; JPEGImages/*.jpg,
    SegmentationClassAug/*.png) layout -> the dataset over them."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataSet, VOCDataSet
    rng = np.random.default_rng(1)
    lines = []
    if style == "voc":
        os.makedirs(os.path.join(root, "JPEGImages")); os.makedirs(os.path.join(root, "SegmentationClassAug"))
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        img, lab = rng.integers(0, 256, (h, w, 3), dtype=np.uint8), rng.integers(0, 21, (h, w), dtype=np.uint8)
        if style == "voc":
            cv2.imwrite(os.path.join(root, "JPEGImages", "im%02d.jpg" % i), img)
            cv2.imwrite(os.path.join(root, "SegmentationClassAug", "im%02d.png" % i), lab)
            lines.append("im%02d" % i)
        else:
            cv2.imwrite(os.path.join(root, "i%02d.png" % i), img); cv2.imwrite(os.path.join(root, "l%02d.png" % i), lab)
            lines.append("i%02d.png l%02d.png" % (i, i))
    with open(os.path.join(root, "train.lst"), "w") as f:
        f.write("\n".join(lines) + "\n")
    cls = VOCDataSet if style == "voc" else CSDataSet
    return cls(str(root), os.path.join(str(root), "train.lst"), crop_size=(32, 48), mean=(104.0, 117.0, 123.0), scale=True, mirror=True)


def _raw(batch):
    images, labels, augs, sizes, names = batch
    images = images if isinstance(images, list) else list(images)
    return list(names), augs.clone(), [t.clone() for t in images], sizes.clone()


def _same_raw(a, b):
    return a[0] == b[0] and torch.equal(a[1], b[1]) and all(torch.equal(x, y) for x, y in zip(a[2], b[2])) and torch.equal(a[3], b[3])


@pytest.mark.parametrize("workers", [0, 3])
@pytest.mark.parametrize("style", ["cityscapes", "voc"])
def test_loader_resumes_the_interrupted_iteration(tmp_path, style, workers):
    """After load_state_dict at batch k, the loader yields batches k.. of the uninterrupted iteration: the same names, files and
    augmentation draws.  Shuffled, mixed image sizes, every k."""
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader
    ds = _write_dataset(tmp_path, style)
    mk = lambda: CSDataLoader(ds, batch_size=2, shuffle=True, num_workers=workers, pin_memory=False)   # noqa: E731
    torch.manual_seed(11); random.seed(12); np.random.seed(13)
    full, states = [], {}
    loader = mk()
    for i, b in enumerate(loader.host_batches()):
        full.append(_raw(b))
        states[i + 1] = (loader.state_dict(), random.getstate(), np.random.get_state())
    assert len(full) == 6 and len({n for b in full for n in b[0]}) == 11
    assert len({tuple(x.shape) for b in full for x in b[2]}) > 1          # mixed sizes reach the batches
    for k in range(1, 6):
        sd, py, npy = states[k]
        torch.manual_seed(99); random.seed(98); np.random.seed(97)
        if workers == 0:                                                  # the draws come from this process's generators
            random.setstate(py); np.random.set_state(npy)
        again = mk()
        again.load_state_dict(sd)
        rest = [_raw(b) for b in again.host_batches()]
        assert len(rest) == 6 - k, (k, len(rest))
        assert all(_same_raw(x, y) for x, y in zip(rest, full[k:])), k
        assert again.state_dict()["batches"] == 6
    # without a loaded position, the iteration is torch's DataLoader's, draw for draw
    torch.manual_seed(11); random.seed(12); np.random.seed(13)
    plain = [_raw(b) for b in mk().loader]
    assert all(_same_raw(x, y) for x, y in zip(plain, full))


def test_loader_state_mismatch_raises(tmp_path):
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader
    ds = _write_dataset(tmp_path, "cityscapes")
    loader = CSDataLoader(ds, batch_size=2, shuffle=True, num_workers=0, pin_memory=False)
    next(iter(loader.host_batches()))
    sd = loader.state_dict()
    for field, v in (("batch_size", 4), ("num_samples", 5), ("shuffle", False), ("num_workers", 2)):
        other = CSDataLoader(ds, batch_size=2, shuffle=True, num_workers=0, pin_memory=False)
        with pytest.raises(ValueError, match=field):
            other.load_state_dict(dict(sd, **{field: v}))
        assert other._resume is None


def test_image_size_reads_headers_like_cv2(tmp_path):
    """PNG (color / gray), baseline and progressive JPEG from the header; another format (BMP) by decoding."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset.datasets import _header_size, image_size
    rng = np.random.default_rng(0)
    for i, (h, w) in enumerate(SIZES):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        files = {"c.png": img, "g.png": img[..., 0], "b.jpg": img, "p.jpg": img, "x.bmp": img}
        for name, a in files.items():
            path = str(tmp_path / ("%d%s" % (i, name)))
            cv2.imwrite(path, a, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if name == "p.jpg" else [])
            want = cv2.imread(path, cv2.IMREAD_COLOR).shape[:2]
            assert tuple(image_size(path)) == want, name
            assert (_header_size(path) is None) == name.endswith(".bmp"), name
