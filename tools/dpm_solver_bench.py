#!/usr/bin/env python
"""DPM_Solver timing on one GPU through the drop-in dpm_solver module, against DDIMSampler: SD1.5 size (ControlNet +
UNet, LoRA rank 128, synthetic weights), batch 4, 512x512 (latent 4x64x64), classifier-free guidance 7.5, batched
CFG and CUDA graphs (`model_wrapper(model.apply_model, ...)`).

    python tools/dpm_solver_bench.py [--reps 3] [--steps 20] [--out FILE]

Reports ms per step (host clock around sample() ending in a device synchronise; median of `reps` runs after one
warm-up run of each configuration, configurations interleaved) for DDIM, 2M++ (multistep order 2, data prediction),
3M++ (multistep order 3) and singlestep-3 (DPM-Solver-fast, noise prediction), every one `steps` model evaluations;
and the time of one launch of the update kernel (order-3 multistep, the most history reads) and of the thresholding
kernel at this latent.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from sampler_bench import BATCH, CFG, LATENT, card, kernel_us  # noqa: E402


def kernels_us():
    from ctrlora_b200 import dpm_schedule, ops
    shape = (BATCH, 4, LATENT, LATENT)
    x, m0, m1, m2, out = (torch.randn(shape, device="cuda") for _ in range(5))
    coef = (0.95, -0.1, 0.05, -0.01, 1.1, 0.9, 0.4, 0.6, 0.0)
    k_lo, k_hi, w = dpm_schedule.quantile_rank(x[0].numel())
    x0 = torch.randn(shape, device="cuda") * 3.
    return {"update_kernel_us": kernel_us(lambda: ops.dpm_solver_update("multistep3", x, m0, coef, m1, m2, out=out)),
            "threshold_kernel_us": kernel_us(lambda: ops.dpm_threshold_(x0, k_lo, k_hi, w, 1e9), launches=500)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpm_solver_bench needs a CUDA device")
    from bench import build_model
    model = build_model("cuda")
    from cldm.ddim_hacked import DDIMSampler
    from ldm.models.diffusion.dpm_solver import dpm_solver as D
    gen = torch.Generator(device="cuda").manual_seed(1)
    mk = lambda *s: torch.randn(s, device="cuda", generator=gen)
    hint = mk(BATCH, 4, LATENT, LATENT)
    cond = {"c_crossattn": [mk(BATCH, 77, 768)], "c_concat": [hint]}
    ucond = {"c_crossattn": [mk(BATCH, 77, 768)], "c_concat": [hint]}
    x_T = mk(BATCH, 4, LATENT, LATENT)
    ns = D.NoiseScheduleVP("discrete", alphas_cumprod=model.alphas_cumprod)
    fn = D.model_wrapper(model.apply_model, ns, guidance_type="classifier-free", condition=cond,
                         unconditional_condition=ucond, guidance_scale=CFG)
    ddim = DDIMSampler(model)
    S = a.steps
    solvers = {"2M++": (True, dict(order=2, method="multistep")), "3M++": (True, dict(order=3, method="multistep")),
               "singlestep-3": (False, dict(order=3, method="singlestep"))}
    runs = {"ddim": lambda: ddim.sample(S, BATCH, (4, LATENT, LATENT), cond, verbose=False, x_T=x_T,
                                        unconditional_guidance_scale=CFG, unconditional_conditioning=ucond, eta=0.0)}
    for name, (px, kw) in solvers.items():
        runs[name] = (lambda px=px, kw=kw: D.DPM_Solver(fn, ns, predict_x0=px).sample(x_T, steps=S, **kw))
    times = {n: [] for n in runs}

    def timed(fn_):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn_()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    with torch.no_grad():
        for fn_ in runs.values():   # warm-up: graph capture, weight caches
            timed(fn_)
        for _ in range(a.reps):
            for n, fn_ in runs.items():
                times[n].append(timed(fn_))
        kern = kernels_us()
    res = {"metric": "dpm_solver_ms_per_step", "gpu": card(), "batch": BATCH, "resolution": 8 * LATENT, "cfg": CFG,
           "steps": S, "config": "ctrlora_finetune_sd15_rank128, synthetic weights, batched CFG, CUDA graphs",
           "reps": a.reps,
           "solvers": [{"solver": n, "ms_per_step": round(1e3 * statistics.median(v) / S, 2),
                        "ms_per_step_min_max": [round(1e3 * min(v) / S, 2), round(1e3 * max(v) / S, 2)]}
                       for n, v in times.items()],
           **{k: round(v, 2) for k, v in kern.items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
