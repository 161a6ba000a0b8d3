"""Training throughput and peak memory with and without gradient accumulation (accumulate_grad_batches = k), CUDA graphs
on, synthetic data at 512x512 (latent 4x64x64):

    python tools/accum_throughput.py [--windows N] [--warmup W]          # one GPU
    torchrun --nproc_per_node 8 tools/accum_throughput.py                 # data-parallel, NCCL

Workloads: finetune rank 128 at micro-batch 16 x k 1 (bench.py's train workload) and 4 x k 4; pretraining (9 tasks,
multi-task schedule) at 8 x k 1, 1 x k 1 and 1 x k 4 (the reference's --bs 1 --gradacc 4 recipe per GPU).  Each is
timed over N optimizer steps (windows) after W warm-up windows, with CUDA events around the timed windows.  Prints one
JSON line: images/s (all GPUs), ms per optimizer step, peak allocated memory of rank 0, the GPU's name and its power
limit read in the same run.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("finetune", 16, 1), ("finetune", 4, 4), ("pretrain", 8, 1), ("pretrain", 1, 1), ("pretrain", 1, 4)]


def gpu_info(index):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(index)],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [c.strip() for c in out.split(",")] if out else (torch.cuda.get_device_name(index), None)
    return {"gpu": name, "power_limit": power}


def run(kind, micro, k, args, rank, world, device):
    import numpy as np
    import torch.distributed as dist
    import bench
    from ctrlora_b200.scheduler import TaskSchedule
    from ctrlora_b200.train import FinetuneTrainer, PretrainTrainer
    cfg = "ctrlora_finetune_sd15_rank128.yaml" if kind == "finetune" else "ctrlora_pretrain_sd15_9tasks_rank128.yaml"
    model = bench.build_model(device, seed=0, config=os.path.join(ROOT, "configs", cfg))
    cls = FinetuneTrainer if kind == "finetune" else PretrainTrainer
    trainer = cls(model, lr=1e-5, accumulate_grad_batches=k)
    gen = torch.Generator().manual_seed(200 + rank)
    L = bench.LATENT
    data = [torch.randn(micro, 4, L, L, generator=gen), torch.randn(micro, 4, L, L, generator=gen),
            torch.randn(micro, bench.CTX_TOKENS, bench.CTX_DIM, generator=gen),
            torch.randint(0, 1000, (micro,), generator=gen), torch.randn(micro, 4, L, L, generator=gen)]
    dev = [v.to(device) for v in data]
    torch.cuda.reset_peak_memory_stats(device)
    trainer.capture(*dev)
    tasks = None
    if kind == "pretrain":
        np.random.seed(1000 + rank)  # a different permutation stream per rank, like the reference's un-seeded ranks
        sched = TaskSchedule(trainer.tasks, largest_dataset_size=max(micro, 8) * 64, batch_size=micro)
        tasks = []
        while len(tasks) < (args.warmup + args.windows) * k:
            tasks += list(sched)
        tasks = iter(tasks)

    def window():
        for _ in range(k):
            loss = trainer.step(*dev) if tasks is None else trainer.step(*dev, task=next(tasks))
        return loss

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        window()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.windows):
        loss = window()
    e1.record()
    barrier()
    t = torch.tensor([e0.elapsed_time(e1)], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = t.item()
    res = {"workload": kind, "micro_batch": micro, "accumulate_grad_batches": k, "batch_per_step": world * micro * k,
           "images_per_sec": world * micro * k * args.windows / (ms / 1e3), "ms_per_optimizer_step": ms / args.windows,
           "peak_mem_gb": torch.cuda.max_memory_allocated(device) / 2 ** 30, "loss": float(loss.item()),
           "step_count": trainer.step_count}
    del trainer, model, dev
    gc.collect()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10, help="timed optimizer steps per workload")
    ap.add_argument("--warmup", type=int, default=3, help="warm-up optimizer steps per workload (after the capture)")
    ap.add_argument("--only", default=None, help="comma-separated subset, e.g. finetune:16:1,pretrain:1:4")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("accum_throughput.py measures on a GPU; none is visible")
    import torch.distributed as dist
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    from ctrlora_b200 import dropin
    dropin.activate()
    todo = WORKLOADS
    if args.only:
        want = {tuple(s.split(":")) for s in args.only.split(",")}
        todo = [w for w in WORKLOADS if (w[0], str(w[1]), str(w[2])) in want]
    results = [run(kind, micro, k, args, rank, world, device) for kind, micro, k in todo]
    if rank == 0:
        line = {"metric": "train_images_per_sec_by_accumulation", "n_gpus": world, "windows": args.windows,
                "warmup": args.warmup, "resolution": 512, "graphs": True, **gpu_info(local_rank), "results": results}
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
