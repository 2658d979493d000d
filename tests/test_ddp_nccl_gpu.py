"""Data-parallel semantics over NCCL on 2 GPUs (utils/parallel.py:54-63,155: loss per GPU on its shard, mean over GPUs):
replicas are identical after construction whatever the per-rank RNG state, the all-reduced flat gradient is the SUM of the
per-rank gradients, and FlatSGD.step applies their MEAN.  Skipped on a machine with fewer than two GPUs."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from oracle import port as oport
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        torch.manual_seed(100 + rank)                                  # DIFFERENT init per rank: NetModel must broadcast rank 0's
        m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world))
        p0 = m.G_solver.flat_p.clone(); d0 = m.D_solver.flat_p.clone()
        gathered = [torch.empty_like(p0) for _ in range(world)]
        dist.all_gather(gathered, p0)
        assert all(torch.equal(g, gathered[0]) for g in gathered), "student replicas differ after construction"
        gathered_d = [torch.empty_like(d0) for _ in range(world)]
        dist.all_gather(gathered_d, d0)
        assert all(torch.equal(g, gathered_d[0]) for g in gathered_d), "discriminator replicas differ after construction"
        u = m.D_model.l1[0].module.weight_u.detach().clone()
        gu = [torch.empty_like(u) for _ in range(world)]
        dist.all_gather(gu, u)
        assert all(torch.equal(g, gu[0]) for g in gu), "spectral-norm vectors differ after construction"
        images, labels = oport.synthetic_batch(1, 512, 512, seed=7 + rank)          # each rank its own shard
        m.set_input((images, labels, None, None))
        for drop in m.student.dropouts():                                           # fixed Dropout2d masks: the two passes below must agree
            drop.injected = (torch.rand(1, 128, generator=torch.Generator().manual_seed(5 + rank)) >= 0.1).float()
        buckets, m.G_solver._buckets = m.G_solver._buckets, None                     # first pass: plain (un-overlapped) exchange
        assert buckets is not None and len(buckets) >= 2
        d_state = {k: v.clone() for k, v in m.D_model.state_dict().items()}         # D(S) advances the spectral-norm vectors / BN stats
        m._student_phase()
        local = m.G_solver.flat_g.clone()
        m.G_solver.all_reduce_grads(world)
        summed = m.G_solver.flat_g.clone()
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        ref_sum = sum(parts)
        err = float((summed - ref_sum).norm() / ref_sum.norm())
        assert err < 1e-6, err
        # second pass over the same weights / inputs with the bucketed all-reduce issued from inside backward (gradients written directly into
        # the flat buffer report themselves; the weight-gradient stream is a producer the NCCL stream waits for): same sums
        m.G_solver._buckets = buckets
        with torch.no_grad():
            for k, v in m.D_model.state_dict().items():
                v.copy_(d_state[k])
        m._student_phase()
        assert m._g_reduced
        torch.cuda.synchronize()
        # same sums (three conv-bias gradients come from an atomicAdd column sum: last-bit differences between two passes are expected)
        err_o = float((m.G_solver.flat_g - summed).norm() / summed.norm())
        assert err_o < 1e-6, (err_o, float((m.G_solver.flat_g - summed).abs().max()))
        lr, mom, wd = m.G_solver.param_groups[0]["lr"], 0.9, m.args.weight_decay
        m.G_solver.step()
        expect = p0 - lr * (ref_sum / world + wd * p0)                               # first step: momentum buffer is zero
        err2 = float((m.G_solver.flat_p - expect).norm() / (lr * (ref_sum / world + wd * p0)).norm())
        assert err2 < 1e-5, err2
        m.discriminator_backward()
        pd = m.D_solver.flat_p.clone()
        gd = [torch.empty_like(pd) for _ in range(world)]
        dist.all_gather(gd, pd)
        assert all(torch.equal(g, gd[0]) for g in gd), "discriminator replicas diverged after one step"
        if rank == 0:
            out.put(("ok", err, err2))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_two_rank_nccl_gradient_average_through_flat_sgd():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_worker, args=(2, 29533, q), nprocs=2, join=True)
    res = q.get(timeout=10)
    print("\nPARITY nccl_dp_world2", res)
    assert res[0] == "ok", res


def _sync_bn_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from structure_knowledge_distillation_b200 import ops
        from structure_knowledge_distillation_b200.libs import InPlaceABNSync
        g = torch.Generator().manual_seed(11)
        N, C, H, W = 4, 96, 9, 13
        x = torch.randn(N, C, H, W, generator=g) * 1.7 + 0.4
        dout = torch.randn(N, C, H, W, generator=g)
        w0, b0 = torch.randn(C, generator=g), torch.randn(C, generator=g) * 0.2

        def run(xs, ds, sync):
            bn = InPlaceABNSync(C, activation="leaky_relu", slope=0.01).cuda().train()
            bn.sync_stats = sync
            with torch.no_grad():
                bn.weight.copy_(w0); bn.bias.copy_(b0)
            xi = ops.to_nhwc(xs.cuda()).requires_grad_(True)
            y = bn(xi)
            y.backward(ops.to_nhwc(ds.cuda()))
            return y.detach(), xi.grad, bn.weight.grad, bn.bias.grad, bn.running_mean.clone(), bn.running_var.clone()
        half = slice(rank * N // world, (rank + 1) * N // world)
        y, dx, dw, db, rm, rv = run(x[half], dout[half], True)                 # this rank's shard, synchronised statistics
        dist.all_reduce(dw); dist.all_reduce(db)                                # parameter gradients: summed over ranks (as the optimizer's exchange does)
        yf, dxf, dwf, dbf, rmf, rvf = run(x, dout, False)                       # the whole batch on one GPU
        rel = lambda a, b: float((a - b).norm() / b.norm().clamp_min(1e-30))
        errs = dict(y=rel(y, yf[half]), dx=rel(dx, dxf[half]), dw=rel(dw, dwf), db=rel(db, dbf), rm=rel(rm, rmf), rv=rel(rv, rvf))
        assert max(errs.values()) < 2e-5, errs
        if rank == 0:
            out.put(("ok", errs))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_sync_bn_two_ranks_equals_full_batch():
    """InPlaceABNSync with sync_stats over 2 NCCL ranks, each holding half of a batch (libs/functions.py:177-209,255-283 semantics:
    combined mean / variance, running statistics with the global count, edz / eydz averaged over ranks) == the whole batch on one GPU:
    outputs, input gradients, summed parameter gradients, running statistics."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_sync_bn_worker, args=(2, 29571, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    assert res[0] == "ok", res
    print("\nPARITY sync_bn_world2", res[1])


def _nvls_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from structure_knowledge_distillation_b200.optim import FlatSGD
        # ---- optimizer level: ragged parameter list, two steps (momentum), against the explicit formula on gathered gradients
        gen = torch.Generator().manual_seed(3)
        shapes = [(64, 3, 3, 3), (64,), (19, 128, 1, 1), (7,), (513, 33), (1,)]
        init = [torch.randn(s, generator=gen) for s in shapes]
        params = [torch.nn.Parameter(t.clone().cuda()) for t in init]
        opt = FlatSGD(params, 0.05, momentum=0.9, weight_decay=5e-4, symmetric=True)
        opt.enable_nvls()
        p_ref = opt.flat_p.clone(); m_ref = torch.zeros_like(p_ref)
        worst = 0.0
        for step in range(2):
            opt.zero_grad()
            g_local = torch.randn(opt.flat_g.shape, generator=torch.Generator().manual_seed(50 + 10 * step + rank)).cuda()
            opt.flat_g.copy_(g_local)
            parts = [torch.empty_like(g_local) for _ in range(world)]
            dist.all_gather(parts, g_local)
            d = sum(parts) / world + 5e-4 * p_ref
            m_ref = 0.9 * m_ref + d
            p_ref = p_ref - 0.05 * m_ref
            opt.step()                                                   # dispatches to step_nvls(): barrier | ld_reduce + SGD + multicast | barrier
            torch.cuda.synchronize()
            worst = max(worst, float((opt.flat_p - p_ref).abs().max() / p_ref.abs().max()))
            allp = [torch.empty_like(p_ref) for _ in range(world)]
            dist.all_gather(allp, opt.flat_p.clone())
            assert all(torch.equal(a, allp[0]) for a in allp), "replicas differ after the multicast store"
        assert worst < 1e-6, worst
        assert torch.equal(params[4].data, opt.flat_p[opt._offsets[4]:opt._offsets[4] + 513 * 33].view(513, 33))   # parameters are views
        sd = opt.state_dict()                                            # momentum is sharded: state_dict() reassembles it
        assert float((sd["momentum"] - m_ref).abs().max() / m_ref.abs().max()) < 1e-6
        # ---- model level: one distillation step with the fused exchange == the same step with NCCL all-reduce + SGD
        from oracle import port as oport
        from structure_knowledge_distillation_b200.networks.kd_model import NetModel
        from structure_knowledge_distillation_b200.utils.train_options import make_args
        res = {}
        for mode in ("nccl", "nvls"):
            torch.manual_seed(100)
            m = NetModel(make_args(batch_size=1, pi=True, pa=True, ho=True, adv_loss_type="hinge", gpu_num=world, allreduce=mode))
            images, labels = oport.synthetic_batch(1, 512, 512, seed=7 + rank)
            m.set_input((images, labels, None, None))
            for drop in m.student.dropouts():
                drop.injected = (torch.rand(1, 128, generator=torch.Generator().manual_seed(5 + rank)) >= 0.1).float()
            m.optimize_parameters()
            torch.cuda.synchronize()
            res[mode] = (m.G_solver.flat_p.clone(), m.D_solver.flat_p.clone())
            del m
        eg = float((res["nvls"][0] - res["nccl"][0]).abs().max() / res["nccl"][0].abs().max())
        ed = float((res["nvls"][1] - res["nccl"][1]).abs().max() / res["nccl"][1].abs().max())
        assert eg < 1e-5 and ed < 1e-5, (eg, ed)
        if rank == 0:
            out.put(("ok", dict(optimizer=worst, model_G=eg, model_D=ed)))
    except Exception as e:                                              # noqa: BLE001
        out.put(("fail", rank, repr(e)))
        raise
    finally:
        dist.destroy_process_group()


def test_nvls_fused_sgd_two_ranks():
    """Gradient exchange fused into the SGD kernel over NVSwitch multicast (skd_sgd_step_nvls: multimem.ld_reduce + multimem.st):
    equals p - lr * (mu * v + mean_over_ranks(g) + wd * p) over two steps, replicas bit-identical, and a whole distillation step equals
    the NCCL path's."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    mp.spawn(_nvls_worker, args=(2, 29591, q), nprocs=2, join=True)
    res = q.get(timeout=30)
    assert res[0] == "ok", res
    print("\nPARITY nvls_fused_sgd_world2", res[1])
