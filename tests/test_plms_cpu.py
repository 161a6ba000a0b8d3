"""PLMS host side without a GPU: the drop-in PLMSSampler's tables, time bookkeeping and per-step scalars
(ctrlora_b200.plms_schedule) are bit-exact against what the unmodified reference's PLMSSampler forms
(tests/golden/tiny_plms_golden.pt, SD1.5 alphas_cumprod), and the sampler imports in overlay mode, refuses what the
reference refuses and fails loudly without a GPU."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from golden_io import load_golden  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def g():
    return load_golden(os.path.join(GOLD, "tiny_plms_golden.pt"))


@pytest.fixture(scope="module")
def model():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    return create_model(os.path.join(GOLD, "tiny_finetune.yaml"))


def sampler_for(model, **kw):
    from ctrlora_b200 import dropin
    dropin.activate()
    from ldm.models.diffusion.plms import PLMSSampler
    return PLMSSampler(model, **kw)


def test_fixture_schedule_is_the_sd15_one(g, model):
    assert torch.equal(g["alphas_cumprod"], model.alphas_cumprod.cpu())


@pytest.mark.parametrize("steps", [1, 2, 4, 5, 20, 50])
def test_tables_and_step_scalars_bit_exact(g, model, steps):
    from ctrlora_b200 import plms_schedule
    ref = g["schedule"][steps]
    s = sampler_for(model)
    s.make_schedule(steps, verbose=False)
    assert np.array_equal(s.ddim_timesteps, ref["ddim_timesteps"])
    assert torch.equal(torch.as_tensor(s.ddim_alphas), ref["ddim_alphas"])
    # a numpy array, float64 except at S = 1, where np.asarray sees only the 0-dim fp32 tensor alphacums[0]
    assert s.ddim_alphas_prev.dtype == ref["ddim_alphas_prev"].dtype == (np.float32 if steps == 1 else np.float64)
    assert np.array_equal(s.ddim_alphas_prev, ref["ddim_alphas_prev"])
    assert torch.equal(torch.as_tensor(s.ddim_sqrt_one_minus_alphas), ref["ddim_sqrt_one_minus_alphas"])
    assert torch.equal(torch.as_tensor(s.ddim_sigmas), ref["ddim_sigmas"])
    plan = plms_schedule.plan(plms_schedule.time_range(s.ddim_timesteps), s.ddim_alphas, s.ddim_alphas_prev,
                              s.ddim_sqrt_one_minus_alphas, s.ddim_sigmas)
    assert len(plan) == len(ref["t"])
    assert [st.t for st in plan] == ref["t"] and [st.t_next for st in plan] == ref["t_next"]
    assert [st.index for st in plan] == list(range(len(plan) - 1, -1, -1))
    for k in ("a_t", "a_prev", "sigma_t", "sqrt_one_minus_at", "sqrt_a_t", "sqrt_a_prev", "dir_coef"):
        assert [getattr(st, k) for st in plan] == ref[k], k


def test_time_range_and_t_next():
    from ctrlora_b200 import plms_schedule
    z = np.zeros(1000)
    one = plms_schedule.plan(plms_schedule.time_range(np.array([1])), z, z, z, z)
    assert [(st.t, st.t_next, st.index) for st in one] == [(1, 1, 0)]   # S = 1: t_next is the step itself
    four = plms_schedule.plan(plms_schedule.time_range(np.array([1, 251, 501, 751])), z, z, z, z)
    assert [(st.t, st.t_next, st.index) for st in four] == [(751, 501, 3), (501, 251, 2), (251, 1, 1), (1, 1, 0)]


def test_steps_not_dividing_1000_fail_like_the_reference(g, model):
    """S = 3 gives the DDIM timesteps 1, 334, 667, 1000; the reference's make_schedule fails on the last one"""
    assert g["schedule"][3] == {"error": "IndexError"}
    with pytest.raises(IndexError):
        sampler_for(model).make_schedule(3, verbose=False)


def test_eta_must_be_zero(model):
    s = sampler_for(model)
    with pytest.raises(ValueError, match="ddim_eta must be 0 for PLMS"):
        s.make_schedule(4, ddim_eta=0.5, verbose=False)
    with pytest.raises(ValueError, match="ddim_eta must be 0 for PLMS"):
        s.sample(4, 1, (4, 16, 16), None, eta=0.5, verbose=False)


def test_overlay_import_and_sample_fails_loudly_without_gpu(model):
    from ctrlora_b200 import dropin
    dropin.activate()
    import ldm.models.diffusion.plms as plms
    assert plms.__file__.startswith(dropin.DROPIN_ROOT)
    s = plms.PLMSSampler(model, schedule="linear")
    cond = {"c_crossattn": [torch.zeros(1, 77, 64)], "c_concat": [torch.zeros(1, 4, 16, 16)]}
    with pytest.raises(RuntimeError, match="CUDA"):
        s.sample(4, 1, (4, 16, 16), cond, verbose=False)


@pytest.mark.parametrize("kw", [dict(score_corrector=object()), dict(quantize_x0=True), dict(dynamic_threshold=0.9),
                                dict(noise_dropout=0.1)])
def test_unsupported_options_raise(model, kw):
    with pytest.raises(NotImplementedError, match="not on the CtrLoRA path"):
        sampler_for(model).sample(4, 1, (4, 16, 16), None, verbose=False, **kw)


def test_v_parameterisation_and_original_steps_raise(model):
    s = sampler_for(model)
    s.make_schedule(4, verbose=False)
    with pytest.raises(NotImplementedError, match="ddim_use_original_steps"):
        s.plms_sampling(None, (1, 4, 16, 16), ddim_use_original_steps=True)
    model.parameterization = "v"
    try:
        with pytest.raises(NotImplementedError, match="v-parameterisation"):
            s.sample(4, 1, (4, 16, 16), None, verbose=False)
    finally:
        model.parameterization = "eps"
