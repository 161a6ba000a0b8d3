"""Gradient-accumulation window bookkeeping on CPU (gloo, world_size 2), host logic only: the used-task exchange once per
window, the window's segments and exchange plan, and no collective on a non-final micro-batch.  The arithmetic is covered
by tests/test_grad_accum_gpu.py."""
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
        from ctrlora_b200.train import PretrainTrainer
        model = create_model(os.path.join(ROOT, "tests", "golden", "tiny_pretrain.yaml"))
        trainer = PretrainTrainer(model, accumulate_grad_batches=2)
        G = trainer.G
        calls = []
        orig = torch.distributed.all_reduce

        def counting(t, *a, **kw):
            calls.append(t.numel())
            return orig(t, *a, **kw)

        torch.distributed.all_reduce = counting
        try:
            window = [["canny", "canny"], ["seg", "canny"]][rank]
            start, first, segs = trainer.begin_micro_batch(window[0])
            res = {"first": (start, first, segs), "after_first": len(calls)}
            start, first, segs = trainer.begin_micro_batch(window[1])
            res["second"] = (start, first)
            res["task_exchange"] = list(calls)
            res["keys"] = [k for _, _, k in segs]
            gen = torch.Generator().manual_seed(100 + rank)
            G.flat_g.copy_(torch.randn(G.numel, generator=gen))
            mine = G.flat_g.clone()
            calls.clear()
            trainer.reduce_gradients([(off, n) for off, n, _ in segs])
            res["grad_exchange"] = sorted(calls) == sorted(n for _, n, _ in segs)
        finally:
            torch.distributed.all_reduce = orig
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        total = sum(gathered)
        res["reduced"] = all(torch.allclose(G.flat_g[o:o + n], total[o:o + n], atol=1e-6) for o, n, _ in segs)
        d_off, d_n = trainer.layout["lora"]["depth"]
        res["depth_untouched"] = torch.equal(G.flat_g[d_off:d_off + d_n], mine[d_off:d_off + d_n])
        # the overlapped form: every element of the window's segments in exactly one bucket's exchange
        trainer.allreduce_cuts = "middle,ib9,ib6,ib3"
        plan = trainer.exchange_plan(segs, [r for _, r in trainer.merged_buckets()])
        flat = sorted(r for ranges in plan for r in ranges)
        covered = [0] * len(segs)
        for off, n in flat:
            hits = [i for i, (so, sn, _) in enumerate(segs) if so <= off and off + n <= so + sn]
            assert len(hits) == 1
            covered[hits[0]] += n
        res["plan_exact"] = all(a[0] + a[1] <= b[0] for a, b in zip(flat, flat[1:])) and \
            covered == [n for _, n, _ in segs]
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_window_segments_plan_and_collectives_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=240) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, r in res.items():
        assert r["first"] == (True, True, None) and r["after_first"] == 0, "a non-final micro-batch issues no collective"
        assert r["second"] == (False, rank == 1)
        assert r["task_exchange"] == [3], "one used-task exchange (a mask over the 3 tasks) per window"
        assert r["keys"] == ["base", "canny", "seg"]
        assert r["grad_exchange"] and r["reduced"] and r["depth_untouched"] and r["plan_exact"]


@pytest.mark.parametrize("k", [0, -1, 1.5, True, "2"])
def test_accumulate_grad_batches_is_validated(k):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ctrlora_b200.train import FinetuneTrainer, PretrainTrainer
    model = create_model(os.path.join(ROOT, "tests", "golden", "tiny_finetune.yaml"))
    with pytest.raises(ValueError):
        FinetuneTrainer(model, accumulate_grad_batches=k)
    with pytest.raises(ValueError):
        PretrainTrainer(model, accumulate_grad_batches=k)
