"""Multi-GPU data parallelism over NCCL (SURVEY.md 8(e)): needs >= 2 visible GPUs , skipped otherwise.

  * the overlapped, bucketed all-reduce of the gradient arena equals the SUM of the ranks' local gradients (fp32, <= 1e-6 rel);
  * N ranks x B images == 1 rank x N*B images for a BatchNorm-free model (ViT): mean-loss gradient = average of the shard
    gradients, so parameters after a step agree;
  * replicas stay bit-identical; the single-graph step (NCCL inside the CUDA graph) equals the eager step.
"""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _vit(seed=0):
    from deeplearning_b200.classification.vision_transformer.vit_model import VisionTransformer

    torch.manual_seed(seed)
    return VisionTransformer(img_size=224, patch_size=16, embed_dim=768, depth=2, num_heads=12, num_classes=16)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from deeplearning_b200.engine.trainer import TrainStep

        B = 8
        g = torch.Generator().manual_seed(11)
        x_all = torch.randn(world * B, 3, 224, 224, generator=g)
        y_all = torch.randint(0, 16, (world * B,), generator=g)
        x, y = x_all[rank * B:(rank + 1) * B].to(dev), y_all[rank * B:(rank + 1) * B].to(dev)
        res = {}
        # ---- (1) local gradients, no communication (world_size=1 arena on this rank)
        m = _vit().to(dev).train()
        tr = TrainStep(m, lr=0.0, momentum=0.0, weight_decay=0.0, world_size=1, broadcast=False)
        tr.step_eager(x, y)
        local = tr.arena.flat_g.clone()
        gathered = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(gathered, local)
        expect_sum = torch.stack(gathered).double().sum(0)
        # ---- (2) overlapped bucketed all-reduce (small buckets: many collectives in flight during the backward pass)
        m2 = _vit().to(dev).train()
        tr2 = TrainStep(m2, lr=0.05, momentum=0.9, weight_decay=5e-5, bucket_mb=4.0)
        before = tr2.arena.flat_p.clone()
        tr2.step_eager(x, y)
        got = tr2.arena.flat_g.double()
        res["allreduce_rel"] = float((got - expect_sum).norm() / expect_sum.norm())
        res["buckets"] = tr2.arena.buckets_launched
        res["p_after_eager"] = tr2.arena.flat_p.clone().cpu()
        # ---- (3) one trailing all-reduce gives the same reduced gradient
        m3 = _vit().to(dev).train()
        tr3 = TrainStep(m3, lr=0.05, momentum=0.9, weight_decay=5e-5, overlap=False)
        tr3.step_eager(x, y)
        res["overlap_vs_single_rel"] = float((tr3.arena.flat_g.double() - got).norm() / got.norm())
        # ---- (4) captured step (NCCL nodes inside the graph) == eager step
        m4 = _vit().to(dev).train()
        tr4 = TrainStep(m4, lr=0.05, momentum=0.9, weight_decay=5e-5, bucket_mb=4.0)
        tr4.capture(x, y)
        assert torch.equal(tr4.arena.flat_p, before)          # capture() is side-effect free
        tr4.step(x, y)
        torch.cuda.synchronize()
        res["graph_vs_eager_rel"] = float((tr4.arena.flat_p.double().cpu() - res["p_after_eager"].double()).norm()
                                          / (res["p_after_eager"].double() - before.double().cpu()).norm())
        res["update_norm"] = float((res["p_after_eager"].double() - before.double().cpu()).norm())
        out[rank] = res
        # a CUDA graph that contains NCCL kernels must be gone before the communicator is destroyed
        del tr4, tr3, tr2, tr
        import gc

        gc.collect()
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(240)
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_nccl_step_equals_single_process_double_batch():
    world, port = 2, _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    r0, r1 = out[0], out[1]
    print({k: v for k, v in r0.items() if not torch.is_tensor(v)})
    assert r0["allreduce_rel"] <= 1e-6 and r1["allreduce_rel"] <= 1e-6, (r0["allreduce_rel"], r1["allreduce_rel"])
    assert r0["buckets"] >= 3                                   # really bucketed
    assert r0["overlap_vs_single_rel"] <= 1e-6
    assert torch.equal(r0["p_after_eager"], r1["p_after_eager"])   # replicas stay bit-identical
    assert r0["graph_vs_eager_rel"] <= 1e-3, r0["graph_vs_eager_rel"]
    # single process, double batch (BN-free model): parameters after the same step
    from deeplearning_b200.engine.trainer import TrainStep

    B = 8
    g = torch.Generator().manual_seed(11)
    x_all = torch.randn(world * B, 3, 224, 224, generator=g).cuda()
    y_all = torch.randint(0, 16, (world * B,), generator=g).cuda()
    m = _vit().cuda().train()
    tr = TrainStep(m, lr=0.05, momentum=0.9, weight_decay=5e-5, world_size=1, broadcast=False)
    before = tr.arena.flat_p.clone().cpu()
    tr.step_eager(x_all, y_all)
    single = tr.arena.flat_p.cpu()
    upd_s, upd_d = (single - before).double(), (r0["p_after_eager"] - before).double()
    rel = float((upd_s - upd_d).norm() / upd_s.norm())
    print(f"2 ranks x {B} vs 1 rank x {2 * B}: relative difference of the parameter update {rel:.3g}")
    assert rel <= 2e-3, rel


# ----------------------------------------------------------------------------------------------------- SyncBatchNorm
def _resnet(seed=0):
    from deeplearning_b200.classification.resnet.models.networks import Bottleneck, ResNet

    torch.manual_seed(seed)
    return ResNet(Bottleneck, [1, 1, 1, 1], num_classes=16)


def _sync_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from deeplearning_b200.engine.trainer import TrainStep

        B = 8
        g = torch.Generator().manual_seed(21)
        x_all = torch.randn(world * B, 3, 64, 64, generator=g)
        y_all = torch.randint(0, 16, (world * B,), generator=g)
        # (every rank's shard has its own mean / scale: local and global statistics differ a lot)
        x_all[B:] = x_all[B:] * 1.5 + 0.5
        x, y = x_all[rank * B:(rank + 1) * B].to(dev), y_all[rank * B:(rank + 1) * B].to(dev)
        res = {}
        # ---- op level (sharp): statistics and the two backward sums of one BatchNorm over the GLOBAL batch
        from deeplearning_b200 import ops

        sync = (dist.group.WORLD, world)
        gg = torch.Generator().manual_seed(5)
        xa = torch.randn(world * 4, 12, 12, 64, generator=gg).to(torch.bfloat16)
        xa[4:] = xa[4:] * 2 + 1
        wa = (torch.randn(128, 64, 3, 3, generator=gg) * 0.05)
        ga = torch.randn(world * 4, 12, 12, 128, generator=gg).to(torch.bfloat16)
        gamma = (torch.rand(128, generator=gg) + 0.5).to(dev)
        beta = (torch.randn(128, generator=gg) * 0.2).to(dev)
        wp = ops.pack_weight(wa.to(dev))
        sl = slice(rank * 4, rank * 4 + 4)

        def finalize(c_stats, rows, sync_):
            rm, rv, nb = torch.zeros(128, device=dev), torch.ones(128, device=dev), torch.zeros((), dtype=torch.long, device=dev)
            co = ops.bn_finalize(c_stats, rows, gamma, beta, 1e-5, 0.1, rm, rv, nb, sync=sync_)
            return co, rm, rv

        c_all, st_all = ops.conv2d_fwd(xa.to(dev), wp, 3, 1, want_stats=True)
        co_all, rm_all, rv_all = finalize(st_all, c_all.numel() // 128, None)
        c_loc, st_loc = ops.conv2d_fwd(xa[sl].to(dev).contiguous(), wp, 3, 1, want_stats=True)
        co_syn, rm_syn, rv_syn = finalize(st_loc, c_loc.numel() // 128, sync)
        ops_err = {}
        for k in ("mean", "invstd", "scale", "shift"):
            ops_err["fwd_" + k] = float((getattr(co_syn, k) - getattr(co_all, k)).abs().max() / getattr(co_all, k).abs().max())
        ops_err["running_var"] = float((rv_syn - rv_all).abs().max())
        dx_all, dg_all, db_all, _ = ops.bn_backward(ga.to(dev), c_all, co_all, relu=True)
        dx_syn, dg_syn, db_syn, _ = ops.bn_backward(ga[sl].to(dev).contiguous(), c_all[sl].contiguous(), co_all, relu=True, sync=sync)
        ops_err["dx"] = float((dx_syn.float() - dx_all[sl].float()).abs().max() / dx_all.float().abs().max())
        ops_err["dgamma"] = float((dg_syn * world - dg_all).abs().max() / dg_all.abs().max())
        ops_err["dbeta"] = float((db_syn * world - db_all).abs().max() / db_all.abs().max())
        # the same sums taken in a dgrad epilogue (conv2d_dgrad(bn_mask=...)) and finished by bn_backward_from_sums
        wd = ops.pack_weight((torch.randn(64, 128, 3, 3, generator=gg) * 0.05).to(dev), mode=1)
        dy = torch.randn(world * 4, 12, 12, 64, generator=gg).to(torch.bfloat16)
        g_full = ops.conv2d_dgrad(dy.to(dev), wd, (12, 12), 3, 1)
        dx2_all, dg2_all, _, _ = ops.bn_backward(g_full, c_all, co_all, relu=True)
        dz, sums = ops.conv2d_dgrad(dy[sl].to(dev).contiguous(), wd, (12, 12), 3, 1, bn_mask=(c_all[sl].contiguous(), co_all))
        dx2_syn, dg2_syn, _ = ops.bn_backward_from_sums(dz, sums, c_all[sl].contiguous(), co_all, sync=sync)
        ops_err["fused_dx"] = float((dx2_syn.float() - dx2_all[sl].float()).abs().max() / dx2_all.float().abs().max())
        ops_err["fused_dgamma"] = float((dg2_syn * world - dg2_all).abs().max() / dg2_all.abs().max())
        res["ops_err"] = ops_err
        for name, convert in (("sync", True), ("local", False)):
            m = _resnet()
            if convert:
                m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)   # others/train_with_DDP/train.py:190
            m = m.to(dev).train()
            tr = TrainStep(m, lr=0.05, momentum=0.9, weight_decay=5e-5)
            before = tr.arena.flat_p.clone()
            tr.step_eager(x, y)
            torch.cuda.synchronize()
            res[name] = (tr.arena.flat_p - before).cpu()
            res[name + "_rm"] = m.bn1.running_mean.detach().cpu().clone()
            res[name + "_rv"] = m.layer1[0].bn2.running_var.detach().cpu().clone()
            del tr, m
        out[rank] = res
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(240)
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sync_batchnorm_two_ranks_equal_one_rank_with_the_whole_batch(monkeypatch):
    """convert_sync_batchnorm (the DDP recipe's default, others/train_with_DDP/train.py:190): 2 ranks x B with SyncBatchNorm
    take the step of 1 rank x 2B with BatchNorm (global statistics, globally centred backward sums, averaged gradients);
    per-rank BatchNorm does not.  Both sides run the plain conv -> BN schedule."""
    world, port = 2, _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_sync_worker, args=(world, port, out), nprocs=world, join=True)
    r0, r1 = out[0], out[1]
    assert torch.equal(r0["sync"], r1["sync"]) and torch.equal(r0["sync_rm"], r1["sync_rm"])   # replicas identical
    from deeplearning_b200.engine.trainer import TrainStep

    monkeypatch.setenv("B200_RESNET_ALGEBRA", "0")
    B = 8
    g = torch.Generator().manual_seed(21)
    x_all = torch.randn(world * B, 3, 64, 64, generator=g)
    y_all = torch.randint(0, 16, (world * B,), generator=g)
    x_all[B:] = x_all[B:] * 1.5 + 0.5
    m = _resnet().cuda().train()
    tr = TrainStep(m, lr=0.05, momentum=0.9, weight_decay=5e-5, world_size=1, broadcast=False)
    before = tr.arena.flat_p.clone()
    tr.step_eager(x_all.cuda(), y_all.cuda())
    single = (tr.arena.flat_p - before).cpu().double()
    rel_sync = float((r0["sync"].double() - single).norm() / single.norm())
    rel_local = float((r0["local"].double() - single).norm() / single.norm())
    rm = m.bn1.running_mean.detach().cpu()
    rv = m.layer1[0].bn2.running_var.detach().cpu()
    print(f"parameter update vs 1 rank x {2 * B}: SyncBatchNorm {rel_sync:.3g}, per-rank BatchNorm {rel_local:.3g}")
    assert torch.allclose(r0["sync_rm"], rm, rtol=1e-4, atol=1e-6), float((r0["sync_rm"] - rm).abs().max())
    assert torch.allclose(r0["sync_rv"], rv, rtol=2e-2, atol=1e-4), float((r0["sync_rv"] - rv).abs().max())
    assert not torch.allclose(r0["local_rm"], rm, rtol=1e-2, atol=1e-3)
    # (different bf16 rounding paths of this tiny random-init network differ by ~0.1-0.3 from each other in their gradients;
    #  the sharp check of every scale factor is the op-level comparison made inside the workers)
    assert rel_sync <= 0.25 and rel_sync <= 0.2 * rel_local, (rel_sync, rel_local)
    print("op level, SyncBatchNorm on 2 ranks vs the whole batch on one:", {k: f"{v:.2g}" for k, v in r0["ops_err"].items()})
    for r in (r0, r1):
        for k, v in r["ops_err"].items():
            assert v <= (2e-2 if k in ("dx", "fused_dx") else 2e-4), (k, v)
