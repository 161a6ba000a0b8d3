"""The drop-in dpm_solver module on the sm_90a kernels against the reference's own module
(tests/golden/dpm_solver_golden.pt, tools/make_dpm_solver_golden.py):
  * every scripted trajectory is bit-identical to the reference's, thresholding included, and calls the model at the
    same times;
  * the adaptive solver takes the same number of model evaluations at the same times to within E's rounding (its sum
    order differs from torch's), x within ADAPTIVE_REL;
  * the kernels one by one against their torch-CPU restatement (tests/test_dpm_solver_module_cpu.CpuKernels), and
    thresholding on the shared-memory and the global-memory paths against torch.quantile;
  * end-to-end samples of the tiny finetune model through `model_wrapper(model.apply_model, ...)` (CUDA graphs,
    batched CFG) within E2E_REL of the reference's CPU samples; graph and eager, batched and sequential CFG agree bit for
    bit; DPM_Solver's 2M++ equals DPMSolverSampler bit for bit; the pretrain and 2-LoRA inference models sample.

Bounds: the error measured on an H100 when the bound was set, plus 20 %, written beside it.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pytestmark = pytest.mark.gpu

from golden_io import load_golden  # noqa: E402
import dpm_solver_cases as cases  # noqa: E402
from test_dpm_solver_module_cpu import CpuKernels  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
ADAPTIVE_REL = 7.5e-7  # norm-relative x error of the scripted adaptive runs (H100: 6.19e-7, adaptive-3-x0)
ADAPTIVE_T = 6.5e-6    # relative error of their model input times (H100: 5.40e-6, adaptive-3-eps)
E2E_REL = 5.9e-3       # norm-relative sample error of the tiny finetune model vs the reference's CPU samples
                       # (H100: 4.92e-3, adaptive-3 at CFG 7.5; 3.31e-3 the worst fixed-step run)
POLICIES = [(True, True), (True, False), (False, True), (False, False)]  # (batched_cfg, use_cuda_graph)


def rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / (ref.norm() + 1e-20)).item()


@pytest.fixture(scope="module")
def g():
    return load_golden(os.path.join(GOLD, "dpm_solver_golden.pt"))


@pytest.fixture(scope="module")
def mod():
    from ctrlora_b200 import dropin
    dropin.activate()
    from ldm.models.diffusion.dpm_solver import dpm_solver
    return dpm_solver


@pytest.mark.parametrize("name", sorted(cases.CASES))
def test_scripted_trajectory_bit_exact(g, mod, name):
    ref = g["trajectories"][name]
    x, t_inputs = cases.run_case(mod, cases.CASES[name], g["sd15_alphas_cumprod"], "cuda")
    assert x.is_cuda and x.dtype == torch.float32
    assert t_inputs == ref["t_inputs"]
    assert torch.equal(x.cpu(), ref["x"])


@pytest.mark.parametrize("name", sorted(cases.ADAPTIVE))
def test_adaptive_same_steps(g, mod, name):
    ref = g["adaptive"][name]
    x, t_inputs = cases.run_case(mod, cases.ADAPTIVE[name], g["sd15_alphas_cumprod"], "cuda")
    assert len(t_inputs) == len(ref["t_inputs"])
    t_err = max(abs(a - b) / max(abs(b), 1e-6) for a, b in zip(t_inputs, ref["t_inputs"]))
    e = rel(x, ref["x"])
    print(f"{name}: nfe {len(t_inputs)}, model time rel err {t_err:.2e}, x rel err {e:.2e}")
    assert t_err < ADAPTIVE_T and e < ADAPTIVE_REL


def _rand(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=gen)


@pytest.mark.parametrize("mode", ["first", "diff", "multistep2", "multistep3", "singlestep3_taylor"])
def test_update_kernel_vs_restatement(mode):
    from ctrlora_b200 import ops
    shape = (3, 4, 24, 24)
    x, m0, m1, m2 = (_rand(shape, s) for s in range(4))
    coef = tuple(float(v) for v in _rand((9,), 9).abs() + 0.1)
    n1 = None if mode == "first" else m1
    n2 = m2 if mode in ("multistep3", "singlestep3_taylor") else None
    ref = CpuKernels.dpm_solver_update(mode, x, m0, coef, n1, n2)
    got = ops.dpm_solver_update(mode, x.cuda(), m0.cuda(), coef, None if n1 is None else n1.cuda(),
                                None if n2 is None else n2.cuda())
    assert torch.equal(got.cpu(), ref)


@pytest.mark.parametrize("model_type", ["noise", "x_start", "v"])
@pytest.mark.parametrize("guidance", ["none", "cfg", "classifier"])
@pytest.mark.parametrize("predict_x0", [False, True])
def test_model_output_kernel_vs_restatement(model_type, guidance, predict_x0):
    from ctrlora_b200 import ops
    shape = (2, 4, 16, 16)
    x, oc, ou, gr = (_rand(shape, s) for s in range(10, 14))
    kw = dict(model_type=model_type, predict_x0=predict_x0, scale=7.5, alpha_w=0.31, sigma_w=0.95, grad_coef=1.7,
              sigma_t=0.83, alpha_t=0.56)
    ou_, gr_ = (ou if guidance == "cfg" else None), (gr if guidance == "classifier" else None)
    ref = CpuKernels.dpm_model_output(x, oc, torch.empty_like(x), out_uncond=ou_, grad=gr_, **kw)
    cu = lambda t: None if t is None else t.cuda()
    got = ops.dpm_model_output(x.cuda(), oc.cuda(), torch.empty(shape, device="cuda"), out_uncond=cu(ou_), grad=cu(gr_),
                               **kw)
    assert torch.equal(got.cpu(), ref)


@pytest.mark.parametrize("shape", [(2, 4, 8, 8), (4, 4, 64, 64), (1, 4, 160, 160), (2, 3, 7, 5)])
def test_threshold_kernel_vs_torch_quantile(shape):
    """64x64x4 is the 512x512 latent (shared memory); 160x160x4 (400 KB) takes the global-memory path"""
    from ctrlora_b200 import dpm_schedule, ops
    x0 = _rand(shape, 20) * 3.
    x0[0, 0, 0, 0] = 50.   # outliers above the quantile
    n = x0[0].numel()
    s = torch.quantile(x0.abs().reshape(shape[0], -1), 0.995, dim=1)
    s = torch.maximum(s, 1.2 * torch.ones_like(s)).reshape(-1, 1, 1, 1)
    ref = torch.clamp(x0, -s, s) / s
    k_lo, k_hi, w = dpm_schedule.quantile_rank(n)
    s_out = torch.empty(shape[0], device="cuda")
    got = ops.dpm_threshold_(x0.cuda().contiguous(), k_lo, k_hi, w, 1.2, s_out=s_out)
    assert torch.equal(s_out.cpu(), s.reshape(-1))
    assert torch.equal(got.cpu(), ref)


def test_adaptive_error_kernel_vs_torch():
    from ctrlora_b200 import ops
    shape = (4, 4, 64, 64)
    xl, xp, xh = _rand(shape, 30), _rand(shape, 31), _rand(shape, 32)
    xh = xl + 0.01 * xh
    ref = CpuKernels.dpm_adaptive_error(xl, xp, xh, 0.0078, 0.05)
    got = ops.dpm_adaptive_error(xl.cuda(), xp.cuda(), xh.cuda(), 0.0078, 0.05)
    e = abs(got.item() - ref.item()) / ref.item()
    print(f"adaptive E: {got.item():.8e} vs torch {ref.item():.8e} (rel {e:.2e})")
    assert e < 1e-5


# ---- end to end on the tiny models

def build(yaml_path, control_shapes, unet_shapes, seed):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from oracle import synth
    model = create_model(yaml_path, init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(control_shapes, seed, "control_model."), strict=True)
    model.model.diffusion_model.load_state_dict(synth.synth_state_dict(unet_shapes, seed, "model.diffusion_model."),
                                                strict=True)
    return model.cuda().eval()


@pytest.fixture(scope="module")
def tiny():
    shapes = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    return build(os.path.join(GOLD, "tiny_finetune.yaml"), shapes["control_shapes"], shapes["unet_shapes"],
                 shapes["seed"])


def tiny_inputs():
    from oracle import synth
    mk = lambda n, s: synth.synth_input(n, s, cases.SEED).cuda()
    B, H = cases.B, 16
    hint, hint2 = mk("hint", (B, 4, H, H)), mk("hint2", (B, 4, H, H))
    return mk("dpm_xT", (B, 4, H, H)), hint, hint2, mk("ctx", (B, 77, 64)), mk("uc_ctx", (B, 77, 64))


def _solve(mod, model, cond, ucond, scale, x_T, predict_x0, kw, batched_cfg=True, use_cuda_graph=True):
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=model.alphas_cumprod)
    fn = mod.model_wrapper(model.apply_model, ns, model_type="noise", guidance_type="classifier-free", condition=cond,
                           unconditional_condition=ucond if scale != 1.0 else None, guidance_scale=scale,
                           batched_cfg=batched_cfg, use_cuda_graph=use_cuda_graph)
    assert fn.eps is not None   # a ControlLDM's bound apply_model takes the graph path
    return mod.DPM_Solver(fn, ns, predict_x0=predict_x0).sample(x_T, **kw)


@pytest.mark.parametrize("name", sorted(cases.E2E))
@pytest.mark.parametrize("scale", cases.E2E_SCALES)
def test_tiny_finetune_vs_reference(g, mod, tiny, name, scale):
    x_T, hint, _, ctx, uc = tiny_inputs()
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    px, kw = cases.E2E[name]
    pols = POLICIES if scale != 1.0 else POLICIES[:2]
    with torch.no_grad():
        outs = {pol: _solve(mod, tiny, cond, ucond, scale, x_T, px, kw, *pol) for pol in pols}
    e = max(rel(o, g["e2e"][(name, scale)]) for o in outs.values())
    print(f"tiny finetune {name} scale {scale}: rel err {e:.2e}")
    assert e < E2E_REL
    if name != "adaptive-3":   # the adaptive step control reads E, whose rounding depends on the eps bits
        for pol in pols[1:]:
            assert torch.equal(outs[pol], outs[pols[0]]), pol


def test_multistep2_equals_dpm_solver_sampler(mod, tiny):
    from ldm.models.diffusion.dpm_solver.sampler import DPMSolverSampler
    x_T, hint, _, ctx, uc = tiny_inputs()
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    with torch.no_grad():
        for steps in (5, 16):
            ref, _ = DPMSolverSampler(tiny).sample(steps, x_T.shape[0], tuple(x_T.shape[1:]), cond, verbose=False,
                                                   x_T=x_T, unconditional_guidance_scale=7.5,
                                                   unconditional_conditioning=ucond)
            got = _solve(mod, tiny, cond, ucond, 7.5, x_T, True,
                         dict(steps=steps, order=2, method="multistep", skip_type="time_uniform"))
            assert torch.equal(got, ref), steps


def test_eager_callable_matches_graph_path(mod, tiny):
    """a lambda around apply_model runs eagerly (dict conditions: one call per half) and gives the same bits"""
    x_T, hint, _, ctx, uc = tiny_inputs()
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    ns = mod.NoiseScheduleVP("discrete", alphas_cumprod=tiny.alphas_cumprod)
    fn = mod.model_wrapper(lambda x, t, c: tiny.apply_model(x, t, c), ns, guidance_type="classifier-free",
                           condition=cond, unconditional_condition=ucond, guidance_scale=7.5)
    assert fn.eps is None
    kw = dict(steps=6, order=3, method="multistep")
    with torch.no_grad():
        eager = mod.DPM_Solver(fn, ns, predict_x0=True).sample(x_T, **kw)
        graph = _solve(mod, tiny, cond, ucond, 7.5, x_T, True, kw, batched_cfg=False, use_cuda_graph=False)
    assert torch.equal(eager, graph)


@pytest.mark.parametrize("kind", ["pretrain", "inference"])
def test_variants_sample(mod, kind):
    shapes = load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))
    model = build(os.path.join(GOLD, f"tiny_{kind}.yaml"), shapes[f"{kind}_control_shapes"], shapes["unet_shapes"],
                  shapes["seed"])
    x_T, hint, hint2, ctx, uc = tiny_inputs()
    if kind == "pretrain":
        cond = {"c_crossattn": [ctx], "c_concat": [hint], "task": "depth"}
        ucond = {"c_crossattn": [uc], "c_concat": [hint], "task": "depth"}
    else:
        model.lora_weights = [0.7, 0.3]
        cond = [{"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [ctx], "c_concat": [hint2]}]
        ucond = [{"c_crossattn": [uc], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint2]}]
    kw = dict(steps=6, order=3, method="singlestep")
    with torch.no_grad():
        outs = [_solve(mod, model, cond, ucond, 7.5, x_T, False, kw, use_cuda_graph=graph) for graph in (True, False)]
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
    assert rel(outs[0], x_T) > 1e-2
