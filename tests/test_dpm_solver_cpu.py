"""DPM-Solver++ host side without a GPU: the schedule and per-step coefficients of ctrlora_b200.dpm_schedule are
bit-exact against the reference's own NoiseScheduleVP / model_wrapper / DPM_Solver objects (tests/golden/tiny_dpm_golden.pt,
SD1.5 alphas_cumprod), and the drop-in DPMSolverSampler imports without a GPU and refuses to sample on one it lacks."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def g():
    return torch.load(os.path.join(GOLD, "tiny_dpm_golden.pt"), weights_only=False)


def f32(v):
    return np.float32(v)


@pytest.mark.parametrize("steps", [4, 5, 10, 16, 20, 25])
def test_schedule_and_coefficients_bit_exact(g, steps):
    from ctrlora_b200 import dpm_schedule
    ref = g["schedule"][steps]
    ns = dpm_schedule.DiscreteVPSchedule(g["sd15_alphas_cumprod"])
    plan = dpm_schedule.multistep_plan(g["sd15_alphas_cumprod"], steps)
    assert len(plan) == steps
    assert [st.order for st in plan] == ref["order"]
    for i, st in enumerate(plan):
        s = torch.tensor([st.t])
        assert st.t == ref["t"][i]
        assert st.model_time == ref["model_time"][i]
        assert st.alpha_s == ref["alpha"][i] and st.sigma_s == ref["sigma"][i]
        assert float(ns.marginal_lambda(s)[0]) == ref["lambda"][i]
        assert st.c_x == ref["c_x"][i]
        assert f32(-f32(st.c_m)) == f32(ref["neg_c_m"][i])
        if st.order == 2:
            assert f32(-(f32(st.c_d) * f32(st.inv_r0))) == f32(ref["neg_c_d_inv_r0"][i])


def test_model_times_are_fractional(g):
    """what the int64 embedding used to truncate: for 20 steps every model time after the first is off the integers"""
    times = g["schedule"][20]["model_time"]
    assert times[0] == 999.0
    assert all(t != int(t) for t in times[1:])


def test_step_orders():
    from ctrlora_b200 import dpm_schedule
    assert dpm_schedule.step_orders(3) == [1, 2, 1]
    assert dpm_schedule.step_orders(14)[-1] == 1
    assert dpm_schedule.step_orders(15) == [1] + [2] * 14
    with pytest.raises(ValueError):
        dpm_schedule.step_orders(1)


def test_dropin_imports_without_gpu_and_sample_fails_loudly():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from ldm.models.diffusion.dpm_solver.sampler import DPMSolverSampler
    model = create_model(os.path.join(GOLD, "tiny_finetune.yaml"))
    sampler = DPMSolverSampler(model)
    assert sampler.alphas_cumprod.dtype == torch.float32 and sampler.alphas_cumprod.device == model.device
    cond = {"c_crossattn": [torch.zeros(1, 77, 64)], "c_concat": [torch.zeros(1, 4, 16, 16)]}
    with pytest.raises(RuntimeError, match="CUDA"):
        sampler.sample(4, 1, (4, 16, 16), cond, verbose=False)
