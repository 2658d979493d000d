"""GPU: data-parallel partitioning of CSDataLoader on the device, and sharded evaluation.  The W partitioned loaders' device batches
(augmented images and labels), concatenated, are the one-rank loader's batch of W times the size; evaluate_main over two gloo ranks
sharing one GPU returns, on both ranks, the IU of one process over the whole list, and writes the same prediction PNGs; with two
GPUs (skipped otherwise), SegModel steps fed by partitioned loaders over NCCL keep identical replicas on disjoint samples and the
evaluation reduces on the device."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASSES = 19
CROP = (64, 96)
VAL_SIZES = [(64, 96), (60, 90), (50, 96), (64, 81), (33, 47)]


class _ToyNet(torch.nn.Module):
    """class scores at 1/8 resolution from plain torch ops: the evaluation kernels and the reduction are what is under test.  It
    reads the first three channels, so it also takes the padded 4-channel NHWC images zoom_image makes for the multi-scale pass."""

    def __init__(self, classes=CLASSES):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.w = torch.nn.Parameter(torch.randn(classes, 3, 1, 1, generator=g))

    def forward(self, x):
        return [F.conv2d(F.avg_pool2d(x[:, :3], 8, 8, ceil_mode=True), self.w)]


def write_val_set(root, n=9):
    """`n` Cityscapes-layout image / label pairs no larger than CROP, so an unscaled, unmirrored crop takes the whole image (offset 0
    whatever the draw) -> the dataset."""
    import cv2
    rng = np.random.default_rng(4)
    lines = []
    for i in range(n):
        h, w = VAL_SIZES[i % len(VAL_SIZES)]
        cv2.imwrite(os.path.join(root, "i%02d.png" % i), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        cv2.imwrite(os.path.join(root, "l%02d.png" % i), rng.integers(0, 34, (h, w), dtype=np.uint8))
        lines.append("i%02d.png l%02d.png" % (i, i))
    with open(os.path.join(root, "val.lst"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return val_set(root)


def val_set(root):
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataSet
    return CSDataSet(root, os.path.join(root, "val.lst"), crop_size=CROP, scale=False, mirror=False, mean=(104.0, 117.0, 123.0))


# evaluate_main settings: sliding tiles, whole image, whole image at two scales with the mirrored pass
EVALS = {"sliding": dict(whole=False), "whole": dict(whole=True), "whole_ms_flip": dict(whole=True, scales=(0.75, 1.0), flip=True)}


@pytest.mark.parametrize("W,b", [(2, 2), (3, 1), (3, 2)])
@pytest.mark.parametrize("style", ["cityscapes", "voc"])
def test_device_batches_concatenate_to_the_wide_batch(tmp_path, style, W, b):
    pytest.importorskip("cv2")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_rank_partition_cpu import _write_dataset
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader
    ds = _write_dataset(str(tmp_path), style, 13)
    mk = lambda bs, r, w: CSDataLoader(ds, batch_size=bs, shuffle=True, num_workers=2, drop_last=True, rank=r, world_size=w, seed=6)  # noqa: E731
    wide = [(i.clone(), l.clone(), n) for i, l, _, n in mk(W * b, 0, 1)]
    parts = [[(i.clone(), l.clone(), n) for i, l, _, n in mk(b, r, W)] for r in range(W)]
    assert len(wide) == 13 // (W * b) and all(len(p) == len(wide) for p in parts)
    for g, (images, labels, names) in enumerate(wide):
        assert torch.equal(torch.cat([p[g][0] for p in parts]), images), g
        assert torch.equal(torch.cat([p[g][1] for p in parts]), labels), g
        assert sum((p[g][2] for p in parts), []) == names
    assert wide[0][0].is_cuda and wide[0][1].dtype == torch.int64


_SHARDED = textwrap.dedent('''
    import json, os, sys, numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    sys.path.insert(0, os.path.join(%r, "tests"))
    from test_rank_partition_gpu import _ToyNet, val_set, EVALS, CLASSES
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)                                         # both ranks share the one GPU
    dist.init_process_group("gloo", rank=rank, world_size=world)
    root, out = sys.argv[1], sys.argv[2]
    net = _ToyNet().cuda()
    res = {}
    for name, kw in EVALS.items():
        loader = CSDataLoader(val_set(root), batch_size=1, rank=rank, world_size=world)
        m, iu = evaluate_main(net, loader, 0, "64,96", CLASSES, png_dir=os.path.join(out, name), **kw)
        mine = [(i.clone(), l.clone(), s, n) for i, l, s, n in CSDataLoader(val_set(root), batch_size=1, rank=rank, world_size=world)]
        m2, iu2 = evaluate_main(net, mine, 0, "64,96", CLASSES, distributed=True, **kw)      # a caller's own shards
        assert np.array_equal(iu, iu2) and m == m2
        res[name] = dict(mean=float(m), iu=[float(x) for x in iu], scored=[n for _, _, _, names in mine for n in names])
    with open(os.path.join(out, "rank%%d.json" %% rank), "w") as f:
        json.dump(res, f)
    dist.barrier(); dist.destroy_process_group()
    print("rank", rank, "ok")
''')


def test_sharded_evaluation_gloo_two_ranks_one_gpu_equals_one_process(tmp_path):
    pytest.importorskip("cv2")
    import json
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    root, out, single = tmp_path / "data", tmp_path / "sharded", tmp_path / "single"
    for d in (root, out, single):
        os.makedirs(d)
    ds = write_val_set(str(root))
    script = tmp_path / "sharded_eval.py"
    script.write_text(_SHARDED % (ROOT, ROOT))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", str(script), str(root), str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    ranks = [json.load(open(out / ("rank%d.json" % k))) for k in range(2)]
    net = _ToyNet().cuda()
    for name, kw in EVALS.items():
        m, iu = evaluate_main(net, CSDataLoader(ds, batch_size=1), 0, "64,96", CLASSES, png_dir=str(single / name), **kw)
        for k in range(2):
            assert ranks[k][name]["iu"] == [float(x) for x in iu] and ranks[k][name]["mean"] == float(m), (name, k)
        assert sorted(ranks[0][name]["scored"] + ranks[1][name]["scored"]) == sorted(f["name"] for f in ds.files)
        assert not set(ranks[0][name]["scored"]) & set(ranks[1][name]["scored"])
        files = sorted(os.listdir(single / name))
        assert len(files) == len(ds.files) and sorted(os.listdir(out / name)) == files
        for f in files:
            assert (single / name / f).read_bytes() == (out / name / f).read_bytes(), (name, f)
    assert 0.0 < float(m) < 1.0


def _nccl_worker(rank, world, port, root, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader, CSDataSet
        from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
        from structure_knowledge_distillation_b200.networks.seg_model import SegModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        torch.manual_seed(0)
        m = SegModel(make_args(batch_size=2, seg_model="resnet18", gpu_num=world))
        train = CSDataSet(root, os.path.join(root, "val.lst"), crop_size=(96, 128), scale=True, mirror=True, mean=(104.0, 117.0, 123.0))
        loader = CSDataLoader(train, batch_size=2, shuffle=True, num_workers=2, drop_last=True, rank=rank, world_size=world, seed=1)
        names = []
        for step, (images, labels, _, batch_names) in enumerate(loader):
            m.set_input((images, labels))
            m.optimize_parameters()
            names += batch_names
        assert step + 1 == len(loader) == 9 // (2 * world)
        seen = [None] * world
        dist.all_gather_object(seen, names)
        assert not set(seen[0]) & set(seen[1]), seen
        p = m.G_solver.flat_p.clone()
        ps = [torch.empty_like(p) for _ in range(world)]
        dist.all_gather(ps, p)
        assert all(torch.equal(x, ps[0]) for x in ps), "replicas diverged"
        val = lambda **kw: CSDataLoader(val_set(root), batch_size=1, **kw)           # noqa: E731
        got = m.evalute_model(m._net, val(rank=rank, world_size=world), 0, "64,96", 19, False)
        local = evaluate_main(m._net, val(), 0, "64,96", 19, whole=False)           # every image on this rank, no reduction
        assert np.array_equal(got[1], local[1]) and got[0] == local[0]
        if rank == 0:
            q.put(("ok", float(got[0])))
    except Exception as e:                                              # noqa: BLE001
        q.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_nccl_two_gpus_train_and_evaluate_on_partitioned_loaders(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    pytest.importorskip("cv2")
    import torch.multiprocessing as mp
    write_val_set(str(tmp_path))
    q = mp.get_context("spawn").Queue()
    mp.spawn(_nccl_worker, args=(2, 29565, str(tmp_path), q), nprocs=2, join=True)
    res = q.get(timeout=10)
    assert res[0] == "ok", res
