"""Resuming a run on the H100: a model trained k steps saves its training state; a second model, built from another seed, loads it and
trains on; every loss after the restart and the whole final state (flat parameters and momentum of both solvers, BN running statistics
and num_batches_tracked, spectral-norm u / v) equal an uninterrupted run bit for bit.  The dropout masks and the WGAN-GP alpha are
drawn, not injected, so the restored random streams decide them.  These runs use overlap_streams=False, where repeated steps are
bit-identical (DESIGN.md §6), and Pa levels below 1 024 pooled nodes (the SIMT path, DESIGN.md §4).  Also: CUDA graphs (saved before
and after the capture, loaded into a captured model), the overlapped streams (state round trip only), CSDataLoader's device batches
and two NCCL ranks."""
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_STEPS, K = 5, 2


def _netmodel(seed, batch=1, **kw):
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(seed)
    kw = dict(dict(pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", pool_scale=0.25, overlap_streams=False), **kw)
    return NetModel(make_args(batch_size=batch, num_steps=100, **kw))


def _segmodel(seed, batch=1, **kw):
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(seed)
    return SegModel(make_args(batch_size=batch, num_steps=100, **dict(dict(overlap_streams=False), **kw)))


def _batches(batch, h, w):
    from oracle import port
    return [port.synthetic_batch(batch, h, w, seed=100 + i) for i in range(N_STEPS)]


def _losses(m):
    if not hasattr(m, "D_solver"):
        return [float(m.G_loss), float(m.mc_G_loss)]
    pa = [float(v) for v in m.pa_G_loss] if isinstance(m.pa_G_loss, list) else [float(m.pa_G_loss)]
    return [float(m.G_loss), float(m.mc_G_loss), float(m.pi_G_loss), float(m.D_loss)] + pa


def _train(m, batches, steps):
    """The reference's loop over `steps`: poly learning rates, set_input, optimize_parameters -> the losses of each step."""
    out = []
    for i in steps:
        m.adjust_learning_rate(m.args.lr_g, m.G_solver, i)
        if hasattr(m, "D_solver"):
            m.adjust_learning_rate(m.args.lr_d, m.D_solver, i)
        images, labels = batches[i]
        m.set_input((images, labels, None, None))
        m.optimize_parameters()
        torch.cuda.synchronize()
        out.append(_losses(m))
    return out


def _state(m):
    out = {}
    for prefix, module, solver in m._trained():
        out.update({prefix + k: v.detach().clone() for k, v in module.state_dict().items()})
        out[prefix + "flat_p"], out[prefix + "flat_m"] = solver.flat_p.clone(), solver.flat_m.clone()
        out[prefix + "steps"] = torch.tensor(solver.steps)
    return out


def _assert_same_state(a, b):
    assert a.keys() == b.keys()
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, bad[:10]


def _share_teacher(src, dst):
    if hasattr(src, "teacher"):
        dst.teacher.load_state_dict(src.teacher.state_dict())


CASES = {
    "resnet18_pi_pa_ho_wgangp": (_netmodel, dict(), (1, 512, 512)),
    "resnet18_hinge_preprocess2": (_netmodel, dict(adv_loss_type="hinge", preprocess_GAN_mode=2), (1, 512, 512)),
    "espnet_c": (_netmodel, dict(student="espnet_c"), (2, 360, 480)),
    "espnet": (_netmodel, dict(student="espnet"), (2, 360, 480)),
    "mobilenetv2": (_netmodel, dict(student="mobilenetv2"), (2, 360, 480)),
    "resnet18_pa_levels": (_netmodel, dict(lambda_pa=[0.5, 0.0, 1.0, 0.5, 0.5], pool_scale=[0.125, 0.25, 0.25, 0.25, 0.25]), (1, 512, 512)),
    "seg_resnet101": (_segmodel, dict(seg_model="resnet101"), (2, 96, 128)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_resumed_run_equals_uninterrupted_run(tmp_path, name):
    build, kw, (batch, h, w) = CASES[name]
    batches = _batches(batch, h, w)
    path = str(tmp_path / "state.pth")
    a = build(0, batch, **kw)
    torch.manual_seed(1234); torch.cuda.manual_seed(1234); random.seed(1); np.random.seed(2)
    want = _train(a, batches, range(K))
    a.save_training_state(path, K - 1, epoch=0, best_mean_IU=0.25)
    want += _train(a, batches, range(K, N_STEPS))
    final = _state(a)
    b = build(7, batch, **kw)
    _share_teacher(a, b)
    del a
    torch.manual_seed(99); torch.cuda.manual_seed(99)
    assert b.load_training_state(path) == K - 1 and b.args.last_step == K - 1 and b.best_mean_IU == 0.25
    got = _train(b, batches, range(b.args.last_step + 1, N_STEPS))
    print("\nRESUME %s losses after the restart %s" % (name, got))
    assert got == want[K:]
    _assert_same_state(_state(b), final)


def test_cuda_graph_resume_before_and_after_capture(tmp_path):
    """ResNet18 Pi+Pa+Ho wgan-gp with CUDA graphs (2 eager steps, the capture, replays).  Saved before the capture and loaded into a
    fresh model whose schedule then matches (1 eager step, capture, replays); saved after the capture and loaded into a model whose
    graph is already captured, which replays from the restored parameters and random streams (the captured dropout / alpha draws
    follow the restored generator's seed and offset)."""
    batches = _batches(1, 512, 512)
    before, after = str(tmp_path / "before.pth"), str(tmp_path / "after.pth")
    a = _netmodel(0)
    a.enable_cuda_graphs(warmup=2)
    torch.manual_seed(1234); torch.cuda.manual_seed(1234)
    want = _train(a, batches, [0])
    a.save_training_state(before, 0)
    want += _train(a, batches, [1, 2, 3])                  # eager, capture, replay
    assert a._graphs["captured"]
    a.save_training_state(after, 3)
    rng_after = torch.cuda.get_rng_state()
    want += _train(a, batches, [4])
    final = _state(a)

    c = _netmodel(7)
    _share_teacher(a, c)
    c.enable_cuda_graphs(warmup=1)
    torch.cuda.manual_seed(99)
    c.load_training_state(before)
    got = _train(c, batches, [1, 2, 3, 4])
    assert got[0] == want[1] and got[2:] == want[3:]        # the capture step computes no loss of its own
    _assert_same_state(_state(c), final)
    del c

    b = _netmodel(8)
    _share_teacher(a, b)
    b.enable_cuda_graphs(warmup=1)
    torch.cuda.manual_seed(98)
    _train(b, batches[::-1], [0, 1, 2])                   # eager, capture, replay on other batches
    assert b._graphs["captured"]
    b.load_training_state(after)
    assert torch.equal(torch.cuda.get_rng_state(), rng_after)
    assert _train(b, batches, [4]) == want[4:]
    _assert_same_state(_state(b), final)


def test_overlapped_streams_state_round_trip(tmp_path):
    """Default streams (student / teacher / discriminator overlap): what loads equals what was saved, bit for bit, random streams
    included (the steps themselves vary from run to run there, DESIGN.md §6)."""
    batches = _batches(1, 512, 512)
    path = str(tmp_path / "state.pth")
    a = _netmodel(0, overlap_streams=True)
    _train(a, batches, range(K))
    a.save_training_state(path, K - 1)
    saved, rng = _state(a), (torch.get_rng_state(), torch.cuda.get_rng_state())
    b = _netmodel(7, overlap_streams=True)
    torch.cuda.manual_seed(5)
    b.load_training_state(path)
    _assert_same_state(_state(b), saved)
    assert torch.equal(torch.get_rng_state(), rng[0]) and torch.equal(torch.cuda.get_rng_state(), rng[1])


def test_loader_device_batches_after_resume(tmp_path):
    """CSDataLoader (2 workers, shuffled, mixed image sizes): after load_state_dict at batch k, the augmented device batches equal
    batches k.. of the uninterrupted iteration bit for bit."""
    cv2 = pytest.importorskip("cv2")
    from structure_knowledge_distillation_b200.dataset.datasets import CSDataLoader, CSDataSet
    rng = np.random.default_rng(4)
    sizes = [(96, 160), (120, 128), (80, 200), (150, 150)]
    with open(tmp_path / "train.lst", "w") as f:
        for i in range(10):
            h, w = sizes[i % len(sizes)]
            cv2.imwrite(str(tmp_path / ("i%d.png" % i)), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
            cv2.imwrite(str(tmp_path / ("l%d.png" % i)), rng.integers(0, 34, (h, w), dtype=np.uint8))
            f.write("i%d.png l%d.png\n" % (i, i))
    ds = CSDataSet(str(tmp_path), str(tmp_path / "train.lst"), crop_size=(64, 96), mean=(104.0, 117.0, 123.0), scale=True, mirror=True)
    mk = lambda: CSDataLoader(ds, batch_size=2, shuffle=True, num_workers=2)         # noqa: E731
    torch.manual_seed(3)
    loader, full, states = mk(), [], {}
    for i, (images, labels, _, names) in enumerate(loader):
        full.append((images.cpu(), labels.cpu(), names))
        states[i + 1] = loader.state_dict()
    for k in (1, 3):
        torch.manual_seed(77)
        again = mk()
        again.load_state_dict(states[k])
        rest = [(i.cpu(), l.cpu(), n) for i, l, _, n in again]
        assert len(rest) == len(full) - k
        for (gi, gl, gn), (wi, wl, wn) in zip(rest, full[k:]):
            assert gn == wn and torch.equal(gi, wi) and torch.equal(gl, wl)


def _ddp_worker(rank, world, port_no, path, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port_no), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port
        a = _segmodel(100 + rank, seg_model="resnet18")
        torch.cuda.manual_seed(10 + rank)                                  # each rank its own dropout stream
        a.set_input(port.synthetic_batch(1, 128, 128, seed=7 + rank))
        a.optimize_parameters()
        a.save_training_state(path, 0)
        saved, rng = _state(a), torch.cuda.get_rng_state()
        b = _segmodel(200 + rank, seg_model="resnet18")
        torch.cuda.manual_seed(0)
        b.load_training_state(path)
        loaded = _state(b)
        same = all(torch.equal(v, loaded[k]) for k, v in saved.items()) and torch.equal(torch.cuda.get_rng_state(), rng)
        ranks = [None] * world
        dist.all_gather_object(ranks, same)
        if rank == 0:
            out.put(("ok" if all(ranks) else "fail", ranks))
    except Exception as e:                                                  # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_save_and_load(tmp_path):
    """Two NCCL ranks: one file, each rank gets the replicated state and its own CUDA random stream back.  Skipped with fewer than
    two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    q = mp.get_context("spawn").Queue()
    mp.spawn(_ddp_worker, args=(2, 29657, str(tmp_path / "state.pth"), q), nprocs=2, join=True)
    res = q.get(timeout=30)
    print("\nRESUME two ranks", res)
    assert res[0] == "ok", res
