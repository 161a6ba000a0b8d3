"""Un-graphed DDIM step(s) of the bench workload for ncu / per-launch analysis.

    ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv \
        --log-file launches.csv python tools/profile_step.py
    python tools/profile_step.py --gemm-json gemm_shapes.json     # per-GEMM CUDA-event timings

The profiled region (cudaProfilerStart/Stop) is exactly one DDIM step with batched CFG at batch 4.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gemm-json", default=None)
    ap.add_argument("--batch", type=int, default=bench.BATCH)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    from ctrlora_b200 import dropin, ops
    dropin.activate()
    from cldm.ddim_hacked import DDIMSampler
    model = bench.build_model(device)
    sampler = DDIMSampler(model, batched_cfg=True, use_cuda_graph=False)
    sampler.make_schedule(50, ddim_eta=0.0, verbose=False)
    B = args.batch
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 4, 64, 64, generator=g).to(device)
    hint = torch.randn(B, 4, 64, 64, generator=g).to(device)
    ctx = torch.randn(B, 77, 768, generator=g).to(device)
    uc = torch.randn(B, 77, 768, generator=g).to(device)
    cond = {"c_crossattn": [ctx], "c_concat": [hint]}
    ucond = {"c_crossattn": [uc], "c_concat": [hint]}
    ts = torch.full((B,), 981, device=device, dtype=torch.long)
    def step():
        with sampler.run_mode():  # a step inside a sampling run: the text context's K / V^T projections are cached
            return sampler.p_sample_ddim(x, cond, ts, index=49, unconditional_guidance_scale=7.5, unconditional_conditioning=ucond)

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    if args.gemm_json:
        ops._GEMM_PROFILE = []
        ops._GEMM_SHAPES = []
        step()
        torch.cuda.synchronize()
        recs = [dict(shape, ms=r[1].elapsed_time(r[2]), gflop=r[0] / 1e9) for shape, r in zip(ops._GEMM_SHAPES, ops._GEMM_PROFILE)]
        ops._GEMM_PROFILE = None
        ops._GEMM_SHAPES = None
        for r in recs:
            r["tflops"] = r["gflop"] / r["ms"] if r["ms"] > 0 else 0
        json.dump(recs, open(args.gemm_json, "w"), indent=0)
        tot = sum(r["ms"] for r in recs)
        print(f"{len(recs)} GEMM launches, {tot:.2f} ms, {sum(r['gflop'] for r in recs) / tot:.1f} TFLOP/s average")
        return
    torch.cuda.profiler.start()
    step()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()


if __name__ == "__main__":
    main()
