"""Generate tests/golden/dpm_solver_golden.pt by running the UNMODIFIED reference module
ldm/models/diffusion/dpm_solver/dpm_solver.py (NoiseScheduleVP, model_wrapper, DPM_Solver) on the CPU, through
tools/ref_shims.py.

    python tools/make_dpm_solver_golden.py

  (a) host schedule: time steps of the three skip types, DPM-Solver-fast's orders and outer time steps, and the
      three noise schedules' marginals and inverse_lambda, for the SD1.5 alphas_cumprod;
  (b) scripted trajectories (tests/dpm_solver_cases.py): method x order x predict_x0 x solver type x skip type,
      t_start / t_end, thresholding, denoise_to_zero, guidance and model types, the adaptive solver; the final x and
      the model input time of every call;
  (c) end-to-end samples of the tiny finetune model for tests/dpm_solver_cases.E2E, with and without CFG 7.5.  As in
      tools/make_golden.py's DPM part, guidance is applied by a function around the two apply_model calls, because
      the reference's classifier-free branch `torch.cat`s the cond dicts (dpm_solver.py:308-310).
Two shims, for two places where the reference raises on its own defaults; nothing else is changed:
  * DPM-Solver-fast's schedule calls `torch.cumsum` without `dim` (dpm_solver.py:459-460), a TypeError for the
    'time_uniform' and 'time_quadratic' skip types: while this tool runs, `dim` defaults to 0 (the tensor is 1-D);
  * order-3 multistep with `lower_order_final` and steps < 15 hands the second-order update all three history
    entries (:1066 -> :740), a ValueError: the second-order update is given the newest two, which are what it uses.
Inputs and weights are regenerated from names by oracle/synth.py; running the tool twice gives identical bytes.
"""
import contextlib
import io
import os
import sys
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import synth  # noqa: E402
from tools import ref_shims  # noqa: E402
from tools.make_golden import build_reference  # noqa: E402
import dpm_solver_cases as cases  # noqa: E402
from golden_io import save_golden  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def sd15_alphas_cumprod():
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    betas = make_beta_schedule("linear", 1000, linear_start=0.00085, linear_end=0.012)
    return torch.tensor(np.cumprod(1. - betas, axis=0), dtype=torch.float32)


def host_record(mod, ac):
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=ac)
    dpm = mod.DPM_Solver(lambda x, t: x, ns)
    rec = {"time_steps": {}, "singlestep": {}, "schedules": {}}
    for skip in ("logSNR", "time_uniform", "time_quadratic"):
        for n in (1, 5, 6, 10, 20):
            rec["time_steps"][(skip, n)] = dpm.get_time_steps(skip, ns.T, 1. / ns.total_N, n, "cpu").clone()
        rec["time_steps"][(skip, "partial")] = dpm.get_time_steps(skip, 0.7, 0.05, 6, "cpu").clone()
        for order in (1, 2, 3):
            for steps in (5, 6, 7, 8, 9, 20):
                if skip == "logSNR" and order == 1:
                    continue
                ts, orders = dpm.get_orders_and_timesteps_for_singlestep_solver(steps, order, skip, ns.T,
                                                                                1. / ns.total_N, "cpu")
                rec["singlestep"][(skip, order, steps)] = (ts.clone(), list(orders))
    t = torch.linspace(1e-3, 1., 257)
    lam = torch.linspace(-8., 8., 129)
    for name, sched in (("discrete", ns), ("linear", mod.NoiseScheduleVP("linear")),
                        ("cosine", mod.NoiseScheduleVP("cosine"))):
        tt = t * sched.T
        rec["schedules"][name] = {"t": tt, "log_mean_coeff": sched.marginal_log_mean_coeff(tt),
                                  "alpha": sched.marginal_alpha(tt), "std": sched.marginal_std(tt),
                                  "lambda": sched.marginal_lambda(tt), "lambda_in": lam,
                                  "inverse_lambda": sched.inverse_lambda(lam)}
    return rec


def e2e_record(mod):
    model = build_reference(os.path.join(GOLD, "tiny_finetune.yaml"), cases.SEED)
    model.encode_first_stage = lambda h: h   # the hint is already a latent-sized tensor (as in tools/make_golden.py)
    model.get_first_stage_encoding = lambda h: h
    H = 16
    mk = lambda n, s: synth.synth_input(n, s, cases.SEED)
    x_T, hint = mk("dpm_xT", (cases.B, 4, H, H)), mk("hint", (cases.B, 4, H, H))
    cond = {"c_crossattn": [mk("ctx", (cases.B, 77, 64))], "c_concat": [hint]}
    ucond = {"c_crossattn": [mk("uc_ctx", (cases.B, 77, 64))], "c_concat": [hint]}
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=model.alphas_cumprod.clone().detach().to(torch.float32))
    out = {}
    for name, (px, kw) in cases.E2E.items():
        for scale in cases.E2E_SCALES:
            if scale == 1.0:
                fn = mod.model_wrapper(lambda x, t, c: model.apply_model(x, t, c), ns, model_type="noise",
                                       guidance_type="classifier-free", condition=cond, unconditional_condition=None,
                                       guidance_scale=1.0)
            else:
                def guided(x, t):
                    e_c, e_u = model.apply_model(x, t, cond), model.apply_model(x, t, ucond)
                    return e_u + scale * (e_c - e_u)
                fn = mod.model_wrapper(guided, ns, model_type="noise", guidance_type="uncond")
            log = io.StringIO()
            with torch.no_grad(), contextlib.redirect_stdout(log):
                x = mod.DPM_Solver(fn, ns, predict_x0=px).sample(x_T.clone(), **kw)
            out[(name, scale)] = x
            print(name, scale, log.getvalue().strip())
    return out


def _cumsum(real):
    return lambda input, dim=0, **kw: real(input, dim, **kw)


def _newest_two(real):
    return lambda self, x, model_prev_list, t_prev_list, t, **kw: real(self, x, model_prev_list[-2:], t_prev_list[-2:],
                                                                       t, **kw)


def main():
    torch.set_num_threads(os.cpu_count())
    mod = ref_shims.reference_module("ldm.models.diffusion.dpm_solver.dpm_solver")
    second = mod.DPM_Solver.multistep_dpm_solver_second_update
    with mock.patch.object(torch, "cumsum", _cumsum(torch.cumsum)), \
            mock.patch.object(mod.DPM_Solver, "multistep_dpm_solver_second_update", _newest_two(second)):
        generate(mod)


def generate(mod):
    ac = sd15_alphas_cumprod()
    g = {"sd15_alphas_cumprod": ac, "host": host_record(mod, ac), "trajectories": {}, "adaptive": {}}
    for name, spec in cases.CASES.items():
        x, t_inputs = cases.run_case(mod, spec, ac, "cpu")
        g["trajectories"][name] = {"x": x, "t_inputs": t_inputs}
    for name, spec in cases.ADAPTIVE.items():
        log = io.StringIO()
        with contextlib.redirect_stdout(log):
            x, t_inputs = cases.run_case(mod, spec, ac, "cpu")
        g["adaptive"][name] = {"x": x, "t_inputs": t_inputs}
        print(name, "nfe", len(t_inputs))
    g["e2e"] = e2e_record(mod)
    out = os.path.join(GOLD, "dpm_solver_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    main()
