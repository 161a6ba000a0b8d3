"""N > 1 host logic on CPU (gloo, world_size 2): the flat trainable-gradient buffer, its single all-reduce and the
replica consistency of the parameter set.  No kernels run here (they need sm_90a); the GPU-side arithmetic is covered
by tests/test_train_gpu.py."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from ctrlora_b200 import dropin
        dropin.activate()
        from cldm.model import create_model
        from ctrlora_b200.train import FinetuneTrainer
        torch.manual_seed(0)  # replicas start from identical weights
        model = create_model(os.path.join(ROOT, "tests", "golden", "tiny_finetune.yaml"))
        trainer = FinetuneTrainer(model)
        assert trainer.world == world
        G = trainer.G
        # parameters alias the flat buffer
        p0 = G.params[0]
        G.flat_p[0] = 123.0
        assert p0.reshape(-1)[0].item() == 123.0
        # the overlap buckets partition the flat buffer (every gradient is reduced exactly once), in backward order
        buckets = trainer.gradient_buckets()
        ranges = sorted(r for rs in buckets.values() for r in rs)
        assert ranges[0][0] == 0 and ranges[-1][0] + ranges[-1][1] == G.numel
        assert all(a[0] + a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
        assert all(buckets[k] for k in ("middle", "ib9", "ib6", "ib3", "final"))
        # rank-dependent gradients -> bucket-wise all-reduce == whole-buffer all-reduce
        gen = torch.Generator().manual_seed(100 + rank)
        G.flat_g.copy_(torch.randn(G.numel, generator=gen))
        mine = G.flat_g.clone()
        for k in ("middle", "ib9", "ib6", "ib3", "final"):
            trainer.reduce_gradients(buckets[k])
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        expect = sum(gathered)
        ok = torch.allclose(G.flat_g, expect, atol=1e-6)
        G.flat_g.copy_(mine)
        trainer.reduce_gradients()
        ok = ok and torch.allclose(G.flat_g, expect, atol=1e-6)
        sums = [torch.empty(1) for _ in range(world)]
        dist.all_gather(sums, G.flat_g.sum().reshape(1))
        same = all(torch.equal(sums[0], s) for s in sums)
        q.put((rank, ok, same, G.numel, len(G.names)))
    finally:
        dist.destroy_process_group()


def _pretrain_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from ctrlora_b200 import dropin
        dropin.activate()
        from cldm.model import create_model
        from ctrlora_b200.train import PretrainTrainer
        torch.manual_seed(rank)  # replicas start DIFFERENT (the reference does not seed); rank 0's parameters must win
        model = create_model(os.path.join(ROOT, "tests", "golden", "tiny_pretrain.yaml"))
        trainer = PretrainTrainer(model)
        G = trainer.G
        sums = [torch.empty(1, dtype=torch.float64) for _ in range(world)]
        dist.all_gather(sums, G.flat_p.double().sum().reshape(1))
        synced = all(torch.equal(sums[0], s) for s in sums)
        # ranks train different tasks in the same step (per-rank un-seeded permutation, multi_task_scheduler.py:59)
        task = trainer.tasks[2 * rank]  # rank 0: canny, rank 1: seg; nobody trains depth
        segs = trainer.window_segments([task])
        keys = [k for _, _, k in segs]
        gen = torch.Generator().manual_seed(100 + rank)
        G.flat_g.copy_(torch.randn(G.numel, generator=gen))
        mine = G.flat_g.clone()
        trainer.reduce_gradients([(off, n) for off, n, _ in segs])
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        total = sum(gathered)
        ok = True
        for off, n, _ in segs:
            ok &= torch.allclose(G.flat_g[off:off + n], total[off:off + n], atol=1e-6)
        d_off, d_n = trainer.layout["lora"]["depth"]
        untouched = torch.equal(G.flat_g[d_off:d_off + d_n], mine[d_off:d_off + d_n])
        covered = sum(n for _, n, _ in segs) + d_n == G.numel
        # the bucketed (overlapped) exchange reduces exactly the same elements, once each, in backward order
        trainer.allreduce_cuts = "middle,ib9,ib6,ib3"
        merged = trainer.merged_buckets()
        plan = trainer.exchange_plan(segs, [r for _, r in merged])
        flat = sorted(r for ranges in plan for r in ranges)
        want = sorted((off, n) for off, n, _ in segs)
        disjoint = all(a[0] + a[1] <= b[0] for a, b in zip(flat, flat[1:]))
        same_cover = sum(n for _, n in flat) == sum(n for _, n in want) and flat[0][0] == 0 and \
            all(any(w[0] <= off and off + n <= w[0] + w[1] for w in want) for off, n in flat)
        G.flat_g.copy_(mine)
        for ranges in plan:
            for off, n in ranges:
                dist.all_reduce(G.flat_g[off:off + n])
        bucketed_ok = all(torch.allclose(G.flat_g[off:off + n], total[off:off + n], atol=1e-6) for off, n, _ in segs) and \
            torch.equal(G.flat_g[d_off:d_off + d_n], mine[d_off:d_off + d_n])
        covered = covered and disjoint and same_cover and bucketed_ok and [st for st, _ in merged][-1] == "final" and len(plan) == 5
        q.put((rank, synced, keys, ok, untouched, covered))
    finally:
        dist.destroy_process_group()


def test_pretrain_window_segments_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_pretrain_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=240) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, synced, keys, ok, untouched, covered in res:
        assert synced, "construction-time broadcast of rank 0's parameters"
        assert keys == ["base", "canny", "seg"], keys
        assert ok and untouched and covered


def test_flat_gradient_allreduce_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=240) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok, same, numel, n in res:
        assert ok and same, (rank, ok, same)
        assert n == 246  # LoRA 164 + zero-convs 26 + norms 56 tensors, like the reference's optimizer (SURVEY.md §8a17)
    assert res[0][3] == res[1][3]
