"""CPU: CSDataLoader partitioned over data-parallel ranks (rank / world_size / seed).  On the raw batches the workers return
(`host_batches()`: names, files and augmentation draws, all made on the CPU): the W ranks' batch g, concatenated in rank order, is
batch g of the one-rank loader with W times the batch size; the ranks' shares are disjoint and cover the list; the order and the
draws are keyed by (seed, iteration, position) and leave the process's random streams alone; an interrupted iteration resumes,
also through StepModel's training state on a gloo world of two."""
import os
import random
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(40, 60), (52, 71), (33, 47), (64, 96), (45, 45), (70, 38)]


def _write_dataset(root, style, n):
    """`n` image / label pairs of mixed sizes in the Cityscapes (PNG list) or VOC (JPEG / PNG by name) layout -> the dataset."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataSet, VOCDataSet
    rng = np.random.default_rng(2)
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


@pytest.fixture(scope="module")
def datasets(tmp_path_factory):
    made = {}

    def get(style, n):
        if (style, n) not in made:
            made[style, n] = _write_dataset(tmp_path_factory.mktemp("%s%d" % (style, n)), style, n)
        return made[style, n]
    return get


def _loader(ds, **kw):
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader
    kw.setdefault("shuffle", True)
    return CSDataLoader(ds, pin_memory=False, **kw)


def _raw(batch):
    images, labels, augs, sizes, names = batch
    images = images if isinstance(images, list) else list(images)
    return list(names), augs.clone(), [t.clone() for t in images], sizes.clone()


def _iteration(loader):
    return [_raw(b) for b in loader.host_batches()]


@pytest.mark.parametrize("drop_last", [True, False])
@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("n", [12, 13])
@pytest.mark.parametrize("b", [1, 2])
@pytest.mark.parametrize("W", [1, 2, 3])
@pytest.mark.parametrize("style", ["cityscapes", "voc"])
def test_ranks_concatenate_to_the_wide_batch(datasets, style, W, b, n, workers, drop_last):
    """12 samples fill every W*b here, 13 leave a partial global batch (but for W*b = 1)."""
    ds = datasets(style, n)
    wide = _iteration(_loader(ds, batch_size=W * b, num_workers=workers, drop_last=drop_last, rank=0, world_size=1, seed=7))
    loaders = [_loader(ds, batch_size=b, num_workers=workers, drop_last=drop_last, rank=r, world_size=W, seed=7) for r in range(W)]
    parts = [_iteration(x) for x in loaders]
    for r in range(W):
        assert len(parts[r]) == len(loaders[r]), (r, len(parts[r]), len(loaders[r]))
        assert all(len(p[0]) == b for p in parts[r][:-1])
    assert len(wide) == max(len(p) for p in parts)
    for g, whole in enumerate(wide):
        share = [p[g] for p in parts if g < len(p)]
        assert sum((s[0] for s in share), []) == whole[0], g
        assert torch.equal(torch.cat([s[1] for s in share]), whole[1]), g
        assert all(torch.equal(x, y) for x, y in zip(sum((s[2] for s in share), []), whole[2])), g
        assert torch.equal(torch.cat([s[3] for s in share]), whole[3]), g
    names = [name for p in parts for batch in p for name in batch[0]]
    assert len(names) == len(set(names))                                   # disjoint (the list's names are distinct)
    if drop_last:
        assert len({len(x) for x in loaders}) == 1 and len(loaders[0]) == n // (W * b)
        assert len(names) == n - n % (W * b)
    else:
        assert sorted(names) == sorted(f["name"] for f in ds.files)        # every sample once


def test_order_is_keyed_by_seed_and_iteration_and_leaves_global_streams_alone(datasets):
    from structure_knowledge_distillation_b200.dataset.datasets import partition_order
    ds = datasets("cityscapes", 13)
    names = lambda it: [n for batch in it for n in batch[0]]               # noqa: E731
    torch.manual_seed(1); random.seed(2); np.random.seed(3)
    before = (torch.get_rng_state(), random.getstate(), np.random.get_state())
    a = _loader(ds, batch_size=2, num_workers=0, rank=1, world_size=2, seed=4)
    a0, a1 = _iteration(a), _iteration(a)
    assert torch.equal(torch.get_rng_state(), before[0]) and random.getstate() == before[1]
    npst = np.random.get_state()
    assert np.array_equal(npst[1], before[2][1]) and npst[2:] == before[2][2:]
    torch.manual_seed(10); random.seed(20); np.random.seed(30)             # other process streams: the same batches
    b = _loader(ds, batch_size=2, num_workers=2, rank=1, world_size=2, seed=4)
    b0, b1 = _iteration(b), _iteration(b)
    for x, y in zip(a0 + a1, b0 + b1):
        assert x[0] == y[0] and torch.equal(x[1], y[1])
    assert names(a0) != names(a1)                                          # the next iteration, another order
    c0 = _iteration(_loader(ds, batch_size=2, num_workers=0, rank=1, world_size=2, seed=5))
    assert names(c0) != names(a0)                                          # another seed, another order
    assert partition_order(13, 4, 0) == partition_order(13, 4, 0) != partition_order(13, 5, 0) != partition_order(13, 4, 1)
    assert sorted(partition_order(13, 4, 0)) == list(range(13)) and partition_order(13, 4, 0, shuffle=False) == list(range(13))


def test_unshuffled_single_image_batches_go_round_robin(tmp_path, datasets):
    """The evaluation setting: batch 1, no shuffle, drop_last=False -- rank r gets samples r, r + W, ...; the test splits too."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataTestSet, VOCDataTestSet
    ds = datasets("cityscapes", 13)
    for W in (2, 3):
        for r in range(W):
            loader = _loader(ds, batch_size=1, shuffle=False, num_workers=0, rank=r, world_size=W)
            got = [n for batch in loader.host_batches() for n in batch[4]]
            assert got == [ds.files[i]["name"] for i in range(r, 13, W)] and len(loader) == len(got)
    img = np.zeros((8, 8, 3), np.uint8)
    os.makedirs(tmp_path / "JPEGImages")
    for i in range(7):
        cv2.imwrite(str(tmp_path / ("t%d.png" % i)), img); cv2.imwrite(str(tmp_path / "JPEGImages" / ("v%d.jpg" % i)), img)
    (tmp_path / "cs.lst").write_text("".join("t%d.png\n" % i for i in range(7)))
    (tmp_path / "voc.lst").write_text("".join("v%d\n" % i for i in range(7)))
    for test, pre in ((CSDataTestSet(str(tmp_path), str(tmp_path / "cs.lst")), "t"), (VOCDataTestSet(str(tmp_path), str(tmp_path / "voc.lst")), "v")):
        for r in range(3):
            loader = _loader(test, batch_size=1, shuffle=False, num_workers=0, rank=r, world_size=3)
            got = [n for _, _, names in loader._partitioned() for n in names]
            assert got == ["%s%d" % (pre, i) for i in range(r, 7, 3)] and len(loader) == len(got)


@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("style", ["cityscapes", "voc"])
def test_partitioned_loader_resumes_the_interrupted_iteration(datasets, style, workers):
    ds = datasets(style, 13)
    mk = lambda: _loader(ds, batch_size=2, num_workers=workers, drop_last=True, rank=1, world_size=2, seed=9)   # noqa: E731
    loader = mk()
    first = _iteration(loader)                                             # iteration 0, run through
    full, states = [], {0: loader.state_dict()}
    for i, batch in enumerate(loader.host_batches()):                      # iteration 1, a state after every batch
        full.append(_raw(batch))
        states[i + 1] = loader.state_dict()
    after = _iteration(loader)                                             # iteration 2
    assert len(full) == 3 and states[1]["iteration"] == 1 and states[1]["version"] == 2
    for k in range(0, 4):
        torch.manual_seed(99); random.seed(98); np.random.seed(97)         # the process's streams do not matter
        again = mk()
        _iteration(again)                                                  # a loader with history of its own
        again.load_state_dict(states[k])
        rest = _iteration(again)
        if k == 0:                                                         # the state after iteration 0: its (empty) rest
            assert rest == [] and _iteration(again)[0][0] == full[0][0]
            continue
        assert len(rest) == 3 - k
        assert all(x[0] == y[0] and torch.equal(x[1], y[1]) and all(torch.equal(p, q) for p, q in zip(x[2], y[2]))
                   for x, y in zip(rest, full[k:])), k
        assert again.state_dict()["batches"] == 3
        nxt = _iteration(again)                                            # then the iteration after the interrupted one
        assert [b[0] for b in nxt] == [b[0] for b in after] and all(torch.equal(x[1], y[1]) for x, y in zip(nxt, after))
    fresh = mk()
    fresh.load_state_dict(mk().state_dict())                               # no iteration had begun: the first one
    assert [b[0] for b in _iteration(fresh)] == [b[0] for b in first]


def test_partitioned_state_mismatch_raises(datasets):
    ds = datasets("cityscapes", 13)
    loader = _loader(ds, batch_size=2, num_workers=0, rank=1, world_size=2, seed=3)
    next(iter(loader.host_batches()))
    sd = loader.state_dict()
    for field, v in (("rank", 0), ("world_size", 3), ("seed", 4), ("drop_last", True), ("batch_size", 4), ("num_samples", 5),
                     ("shuffle", False), ("num_workers", 2), ("version", 1)):
        other = _loader(ds, batch_size=2, num_workers=0, rank=1, world_size=2, seed=3)
        with pytest.raises(ValueError, match=field):
            other.load_state_dict(dict(sd, **{field: v}))
        assert other._resume is None
    plain = _loader(ds, batch_size=2, num_workers=0)
    with pytest.raises(ValueError, match="rank"):                         # a partitioned position into an unpartitioned loader
        plain.load_state_dict(sd)
    assert "rank" not in plain.state_dict() and plain.state_dict()["version"] == 1
    for bad in (dict(rank=0), dict(world_size=2), dict(rank=2, world_size=2), dict(rank=0, world_size=0), dict(rank=0, world_size=1, seed=-1),
                dict(rank=0.0, world_size=1)):
        with pytest.raises(ValueError, match="rank"):
            _loader(ds, batch_size=2, **bad)


_GLOO = textwrap.dedent('''
    import os, sys, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    sys.path.insert(0, os.path.join(%r, "tests"))
    from test_resume_cpu import _standin
    from test_rank_partition_cpu import _write_dataset, _loader, _raw
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    path, root = sys.argv[1], sys.argv[2]
    if rank == 0:
        _write_dataset(root, "cityscapes", 13)
    dist.barrier()
    import pytest
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataSet
    ds = CSDataSet(root, os.path.join(root, "train.lst"), crop_size=(32, 48), mean=(104.0, 117.0, 123.0))
    mk = lambda: _loader(ds, batch_size=2, num_workers=2, drop_last=True, rank=rank, world_size=world, seed=21)
    loader = mk()
    full = [_raw(b) for b in loader.host_batches()]
    loader = mk()
    it = loader.host_batches()
    next(it)
    m = _standin(seed=0); m.world = world
    m.save_training_state(path, 1, loader=loader)
    d = _standin(seed=1); d.world = world
    again = mk()
    assert d.load_training_state(path, loader=again) == 1
    rest = [_raw(b) for b in again.host_batches()]
    assert len(rest) == len(full) - 1 == 2
    assert all(x[0] == y[0] and torch.equal(x[1], y[1]) for x, y in zip(rest, full[1:]))
    mine = [n for b in full for n in b[0]]
    other = [None] * world
    dist.all_gather_object(other, mine)
    assert not set(other[0]) & set(other[1])
    dist.barrier(); dist.destroy_process_group()
    print("rank", rank, "ok")
''')


def test_partitioned_loader_state_round_trips_through_training_state_gloo_world2(tmp_path):
    """Each of two gloo ranks stops after one batch of its share, saves the training state with its loader, and a fresh loader
    loaded through load_training_state yields the rest of that rank's share."""
    pytest.importorskip("cv2")
    script = tmp_path / "partition_ddp.py"
    script.write_text(_GLOO % (ROOT, ROOT))
    os.makedirs(tmp_path / "data")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29561", str(script), str(tmp_path / "state.pth"), str(tmp_path / "data")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("ok") == 2


def test_sharded_evaluation_needs_a_process_group():
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    import torch.distributed as dist
    assert not dist.is_initialized()
    with pytest.raises(ValueError, match="process group"):
        evaluate_main(torch.nn.Linear(1, 1), [], 0, "64,96", 19, distributed=True)
