"""The drop-in dpm_solver module without a GPU, against the reference's own module run on the CPU
(tests/golden/dpm_solver_golden.pt, tools/make_dpm_solver_golden.py):
  * the three noise schedules, the time steps of the three skip types and DPM-Solver-fast's orders and outer steps are
    bit-exact;
  * every scripted trajectory (method x order x predict_x0 x solver type x skip type, partial runs, thresholding,
    denoise_to_zero, guidance, model types, the adaptive solver) is bit-exact when the four kernels are replaced by a
    torch-CPU restatement of their arithmetic (`CpuKernels`, one torch op per rounding of the kernel).  This pins every
    host scalar and every expression tree the kernels evaluate; tests/test_dpm_solver_module_gpu.py pins the kernels;
  * the module imports without a GPU, CPU tensors fail loudly and the reference's ValueErrors are raised.
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from golden_io import load_golden  # noqa: E402
import dpm_solver_cases as cases  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def g():
    return load_golden(os.path.join(GOLD, "dpm_solver_golden.pt"))


@pytest.fixture(scope="module")
def mod():
    from ctrlora_b200 import dropin
    dropin.activate()
    from ldm.models.diffusion.dpm_solver import dpm_solver
    return dpm_solver


def _f(v):
    return torch.tensor(v, dtype=torch.float32)


def _fma32(a, b, c):
    """fp32 fused multiply-add: the fp32 product is exact in fp64"""
    return torch.from_numpy((a.double() * b.double() + c.double()).numpy().astype(np.float32))


class CpuKernels:
    """ctrlora_b200.ops' DPM-Solver kernels restated with torch CPU ops, one op per rounding of the kernel"""

    @staticmethod
    def dpm_model_output(x, out_cond, m_out, model_type="noise", out_uncond=None, grad=None, predict_x0=False,
                         scale=1.0, alpha_w=1.0, sigma_w=1.0, grad_coef=0.0, sigma_t=1.0, alpha_t=1.0):
        def to_noise(o):
            if model_type == "x_start":
                return (x - _f(alpha_w) * o) / _f(sigma_w)
            if model_type == "v":
                return _f(alpha_w) * o + _f(sigma_w) * x
            return o
        e = to_noise(out_cond)
        if out_uncond is not None:
            u = to_noise(out_uncond)
            e = u + _f(scale) * (e - u)
        if grad is not None:
            e = e - _f(grad_coef) * grad
        if predict_x0:
            e = (x - _f(sigma_t) * e) / _f(alpha_t)
        return m_out.copy_(e)

    @staticmethod
    def dpm_solver_update(mode, x, m0, coef, m1=None, m2=None, out=None):
        a, b, c, d, k0, k1, k2, k3, rd = (_f(v) for v in coef)
        r = a * x - b * m0
        if mode == "diff":
            r = r + c * (m1 - m0)
        elif mode == "multistep2":
            r = r + c * (k0 * (m0 - m1))
        elif mode == "multistep3":
            d10, d11 = k0 * (m0 - m1), k1 * (m1 - m2)
            diff = d10 - d11
            r = (r + c * (d10 + k2 * diff)) + d * (k3 * diff)
        elif mode == "singlestep3_taylor":
            d10, d11 = k0 * (m1 - m0), k1 * (m2 - m0)
            r = (r + c * ((k3 * d10 - k2 * d11) / rd)) + d * ((2. * (d11 - d10)) / rd)
        else:
            assert mode == "first"
        return r

    @staticmethod
    def dpm_threshold_(x0, k_lo, k_hi, weight, max_val, s_out=None):
        v = x0.abs().reshape(x0.shape[0], -1).sort(dim=1).values
        lo, hi, w = v[:, k_lo], v[:, k_hi], _f(weight)
        diff = hi - lo
        q = _fma32(w, diff, lo) if abs(weight) < 0.5 else _fma32(-diff, 1. - w, hi)
        s = torch.maximum(q, _f(max_val)).reshape((-1,) + (1,) * (x0.dim() - 1))
        return x0.copy_(torch.clamp(x0, -s, s) / s)

    @staticmethod
    def dpm_adaptive_error(x_lower, x_prev, x_higher, atol, rtol, err=None):
        delta = torch.max(torch.ones_like(x_lower) * atol, rtol * torch.max(torch.abs(x_lower), torch.abs(x_prev)))
        v = ((x_higher - x_lower) / delta).reshape(x_lower.shape[0], -1)
        return torch.sqrt(torch.square(v).mean(dim=-1, keepdim=True)).max().reshape(1)


@pytest.fixture
def cpu_mod(mod, monkeypatch):
    monkeypatch.setattr(mod, "ops", CpuKernels)
    monkeypatch.setattr(mod, "_check_cuda", lambda *ts: None)
    return mod


def test_noise_schedules_bit_exact(g, mod):
    ac = g["sd15_alphas_cumprod"]
    for name, ref in g["host"]["schedules"].items():
        ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=ac) if name == "discrete" else mod.NoiseScheduleVP(name)
        t = ref["t"]
        assert torch.equal(ns.marginal_log_mean_coeff(t), ref["log_mean_coeff"]), name
        assert torch.equal(ns.marginal_alpha(t), ref["alpha"]), name
        assert torch.equal(ns.marginal_std(t), ref["std"]), name
        assert torch.equal(ns.marginal_lambda(t), ref["lambda"]), name
        assert torch.equal(ns.inverse_lambda(ref["lambda_in"]), ref["inverse_lambda"]), name


def test_time_steps_and_singlestep_orders_bit_exact(g, mod):
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=g["sd15_alphas_cumprod"])
    dpm = mod.DPM_Solver(lambda x, t: x, ns)
    for (skip, n), ref in g["host"]["time_steps"].items():
        got = dpm.get_time_steps(skip, 0.7, 0.05, 6, "cpu") if n == "partial" else \
            dpm.get_time_steps(skip, ns.T, 1. / ns.total_N, n, "cpu")
        assert torch.equal(got, ref), (skip, n)
    for (skip, order, steps), (ts, orders) in g["host"]["singlestep"].items():
        got_ts, got_orders = dpm.get_orders_and_timesteps_for_singlestep_solver(steps, order, skip, ns.T,
                                                                                1. / ns.total_N, "cpu")
        assert got_orders == orders and torch.equal(got_ts, ts), (skip, order, steps)


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_trajectory_with_cpu_kernels_bit_exact(g, cpu_mod, name):
    ref = g["trajectories"][name]
    x, t_inputs = cases.run_case(cpu_mod, cases.CASES[name], g["sd15_alphas_cumprod"], "cpu")
    assert t_inputs == ref["t_inputs"]
    assert torch.equal(x, ref["x"])


@pytest.mark.parametrize("name", sorted(cases.ADAPTIVE))
def test_adaptive_with_cpu_kernels_bit_exact(g, cpu_mod, name):
    ref = g["adaptive"][name]
    x, t_inputs = cases.run_case(cpu_mod, cases.ADAPTIVE[name], g["sd15_alphas_cumprod"], "cpu")
    assert t_inputs == ref["t_inputs"]
    assert torch.equal(x, ref["x"])


def test_cpu_tensors_fail_loudly(mod):
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=torch.linspace(0.999, 0.01, 1000))
    dpm = mod.DPM_Solver(mod.model_wrapper(lambda x, t: torch.zeros_like(x), ns), ns, predict_x0=True)
    x = torch.zeros(1, 4, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        dpm.sample(x, steps=4, order=2, method="multistep")
    with pytest.raises(RuntimeError, match="CUDA"):
        dpm.model_fn(x, torch.ones(1))


def test_reference_errors(mod):
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=torch.linspace(0.999, 0.01, 1000))
    dpm = mod.DPM_Solver(lambda x, t: x, ns)
    with pytest.raises(ValueError, match="noise schedule"):
        mod.NoiseScheduleVP("quadratic")
    with pytest.raises(ValueError, match="skip_type"):
        dpm.get_time_steps("uniform", 1., 1e-3, 5, "cpu")
    with pytest.raises(ValueError, match="order"):
        dpm.get_orders_and_timesteps_for_singlestep_solver(6, 4, "time_uniform", 1., 1e-3, "cpu")
    x = torch.zeros(1, 1)
    with pytest.raises(ValueError, match="order must be 1 or 2 or 3"):
        dpm.singlestep_dpm_solver_update(x, torch.ones(1), torch.ones(1) * 0.5, 4)
    with pytest.raises(ValueError, match="order must be 1 or 2 or 3"):
        dpm.multistep_dpm_solver_update(x, [x], [torch.ones(1)], torch.ones(1) * 0.5, 0)
    with pytest.raises(ValueError, match="solver_type"):
        dpm.singlestep_dpm_solver_second_update(x, torch.ones(1), torch.ones(1) * 0.5, solver_type="euler")
    with pytest.raises(ValueError, match="solver_type"):
        dpm.multistep_dpm_solver_second_update(x, [x, x], [torch.ones(1), torch.ones(1) * 0.7], torch.ones(1) * 0.5,
                                               solver_type="euler")
    with pytest.raises(ValueError, match="adaptive"):
        dpm.dpm_solver_adaptive(x, 1, 1., 1e-3)
    with pytest.raises(ValueError, match="method"):
        dpm.sample(x, method="euler")
    with pytest.raises(AssertionError):
        mod.model_wrapper(lambda x, t: x, ns, model_type="score")
