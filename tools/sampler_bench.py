#!/usr/bin/env python
"""Sampler timing on one GPU: DDIMSampler vs the drop-in DPMSolverSampler and PLMSSampler at SD1.5 size (ControlNet +
UNet, LoRA rank 128, synthetic weights), batch 4, 512x512 (latent 4x64x64), classifier-free guidance 7.5, batched CFG
and CUDA graphs (the samplers' defaults).

    python tools/sampler_bench.py [--reps 3] [--out FILE]

Reports sample() wall time and ms per step (host clock around sample() ending in a device synchronise; median of
`reps` runs after one warm-up run of each configuration, runs of the configurations interleaved), ms per model
evaluation (PLMS evaluates the model S + 1 times in S steps, the others S times), the DPM-Solver++ and PLMS update
kernels' times from CUDA events over many launches, and the card's name and power limit read in the same run.
Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, LATENT, CFG = 4, 64, 7.5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def kernel_us(launch, launches=2000):
    """one launch of `launch`, host dispatch included: CUDA events over `launches` back-to-back launches"""
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def update_kernels_us():
    from ctrlora_b200 import ops
    shape = (BATCH, 4, LATENT, LATENT)
    x, e_c, e_u, m_prev, m_out, o1, o2, o3 = (torch.randn(shape, device="cuda") for _ in range(8))
    dpm = dict(sigma_s=0.9, alpha_s=0.4, c_x=0.95, c_m=-0.1, c_d=-0.05, inv_r0=1.1)
    plms = dict(sqrt_a_t=0.3, sqrt_one_minus_at=0.95, sqrt_a_prev=0.4, dir_coef=0.9)
    return {"dpm_update_kernel_us": kernel_us(lambda: ops.dpm_multistep_update(x, e_c, e_u, m_prev, m_out, CFG, **dpm)),
            # order 4, the steady-state step: the most history reads
            "plms_update_kernel_us": kernel_us(lambda: ops.plms_update(x, e_c, e_u, m_out, CFG, old=(o1, o2, o3),
                                                                       **plms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench needs a CUDA device")
    from bench import build_model
    model = build_model("cuda")
    from cldm.ddim_hacked import DDIMSampler
    from ldm.models.diffusion.dpm_solver.sampler import DPMSolverSampler
    from ldm.models.diffusion.plms import PLMSSampler
    gen = torch.Generator(device="cuda").manual_seed(1)
    mk = lambda *s: torch.randn(s, device="cuda", generator=gen)
    hint = mk(BATCH, 4, LATENT, LATENT)
    cond = {"c_crossattn": [mk(BATCH, 77, 768)], "c_concat": [hint]}
    ucond = {"c_crossattn": [mk(BATCH, 77, 768)], "c_concat": [hint]}
    x_T = mk(BATCH, 4, LATENT, LATENT)
    ddim, dpm, plms = DDIMSampler(model), DPMSolverSampler(model), PLMSSampler(model)
    configs = [("ddim", ddim, 20), ("dpmpp2m", dpm, 20), ("dpmpp2m", dpm, 10), ("plms", plms, 20)]
    evals = lambda n, s: s + 1 if n == "plms" else s
    times = {(n, s): [] for n, _, s in configs}

    def run(sampler, steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sampler.sample(steps, BATCH, (4, LATENT, LATENT), cond, verbose=False, x_T=x_T, unconditional_guidance_scale=CFG,
                       unconditional_conditioning=ucond, eta=0.0)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    with torch.no_grad():
        for _, smp, s in configs:   # warm-up: graph capture, weight caches
            run(smp, s)
        for _ in range(a.reps):
            for n, smp, s in configs:
                times[(n, s)].append(run(smp, s))
        kern = update_kernels_us()
    res = {"metric": "sampler_ms_per_step", "gpu": card(), "batch": BATCH, "resolution": 8 * LATENT, "cfg": CFG,
           "config": "ctrlora_finetune_sd15_rank128, synthetic weights, batched CFG, CUDA graphs", "reps": a.reps,
           "samplers": [{"sampler": n, "steps": s, "sample_s": round(statistics.median(times[(n, s)]), 4),
                         "ms_per_step": round(1e3 * statistics.median(times[(n, s)]) / s, 2),
                         "ms_per_model_eval": round(1e3 * statistics.median(times[(n, s)]) / evals(n, s), 2),
                         "ms_per_step_min_max": [round(1e3 * min(times[(n, s)]) / s, 2),
                                                 round(1e3 * max(times[(n, s)]) / s, 2)]}
                        for n, _, s in configs],
           **{k: round(v, 2) for k, v in kern.items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
