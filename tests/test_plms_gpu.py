"""PLMS on the sm_90a kernels: the fused update kernel `ctrlora_plms_update` at every order against torch, and the
drop-in PLMSSampler against the unmodified reference's PLMSSampler (tests/golden/tiny_plms_golden.pt,
sd15_plms_golden.pt, `tools/make_plms_golden.py`) on every CtrLoRA model kind, under every batched-CFG / CUDA-graph
policy; its loop against a torch restatement of the reference's loop fed the same eps, bit for bit.

Bounds sit about 20 % above what an NVIDIA H100 80GB HBM3 measured, written beside them; the errors are printed under
`pytest -s`."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pytestmark = pytest.mark.gpu

from golden_io import load_golden  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
F64_TOL = 7.5e-7         # update kernel vs fp64 evaluation of the same formula, norm-relative: 6.23e-7 measured (order 4, CFG)
BOUND = {                     # norm-relative error of the final sample vs the reference's
    "tiny_finetune": 3.7e-3,       # 3.04e-3 worst of steps 1 / 4 / 20 with and without CFG (steps 4, CFG 7.5)
    "tiny_intermediates": 4.6e-3,  # 3.81e-3 worst x_inter / pred_x0 entry (steps 4, CFG 7.5)
    "tiny_pretrain": 3.8e-3,       # 3.14e-3 worst task (seg)
    "tiny_inference": 3.7e-3,      # 3.03e-3 (2 LoRAs, weights 0.7 / 0.3)
    "tiny_style": 4.2e-3,          # 3.45e-3 (guess mode; 3.01e-3 with the hint in both halves)
    "sd15": 2.2e-3,                # 1.83e-3 (SD1.5 rank 128, batch 2, steps 20, CFG 7.5)
    # batched vs sequential CFG, same sampler otherwise: fp16 rounding of the two batch layouts; 2.16e-3 at SD1.5
    # (the tiny models measured 0: bit-identical)
    "cfg_policy": 2.6e-3,
}
POLICIES = [(True, True), (True, False), (False, True), (False, False)]  # (batched_cfg, use_cuda_graph)


def rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / (ref.norm() + 1e-20)).item()


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
def g():
    return load_golden(os.path.join(GOLD, "tiny_plms_golden.pt"))


@pytest.fixture(scope="module")
def variants():
    return load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))


@pytest.fixture(scope="module")
def tiny():
    shapes = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    return build(os.path.join(GOLD, "tiny_finetune.yaml"), shapes["control_shapes"], shapes["unet_shapes"], shapes["seed"])


def tiny_inputs(g):
    from oracle import synth
    B, H, seed = g["B"], g["H"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    return dict(x_T=mk("plms_xT", (B, 4, H, H)), hint=mk("hint", (B, 4, H, H)), hint2=mk("hint2", (B, 4, H, H)),
                ctx=mk("ctx", (B, 77, 64)), uc=mk("uc_ctx", (B, 77, 64)), ip=mk("ip", (B, 4, 64)),
                uc_ip=mk("uc_ip", (B, 4, 64)))


def _sample(model, steps, cond, ucond, scale, x_T, batched_cfg=True, use_cuda_graph=True, **kw):
    from ldm.models.diffusion.plms import PLMSSampler
    sampler = PLMSSampler(model, batched_cfg=batched_cfg, use_cuda_graph=use_cuda_graph)
    out, inter = sampler.sample(steps, x_T.shape[0], tuple(x_T.shape[1:]), cond, verbose=False, x_T=x_T,
                                unconditional_guidance_scale=scale, unconditional_conditioning=ucond, **kw)
    assert out.dtype == torch.float32 and out.device == x_T.device
    return out, inter, sampler


def _all_policies(model, steps, cond, ucond, scale, x_T, ref, bound, what, graphed):
    """Samples under every (batched_cfg, use_cuda_graph) policy against `ref`.  `graphed` says whether the conditioning
    takes DDIMSampler's graph path at all: only dicts of tensor lists do (DDIMSampler._flat_cond).  A list of dicts
    (multi-LoRA inference) or a string entry (the pretrain `task`) runs apply_model eagerly under every policy, and
    there the graph-replay == eager check below compares two eager runs."""
    outs = {}
    with torch.no_grad():
        for pol in POLICIES:
            outs[pol], _, sampler = _sample(model, steps, cond, ucond, scale, x_T, *pol)
            assert (sampler.eps_model._graph is not None) == (graphed and pol[1]), pol
    err = max(rel(o, ref) for o in outs.values())
    print(f"{what}: rel err {err:.2e} vs the reference")
    assert err < bound
    for batched in (True, False):
        assert torch.equal(outs[(batched, True)], outs[(batched, False)])   # graph replay == eager, bit for bit
    return outs


# ------------------------------------------------------------------------------------------------ the update kernel
def _torch_update(x, ec, eu, en, old, scale, st, dtype):
    """plms.py:184-244 as torch evaluates it on CUDA tensors in fp32, or the same formula in fp64 with true divisions
    and square roots.  In fp32 the per-step scalars a_t.sqrt(), a_prev.sqrt() and (1 - a_prev - sigma_t**2).sqrt() are
    the host's, torch CPU fp32: the reference's values as run on a CPU (test_plms_cpu.py).  They are not formed on the
    device here because torch's CPU sqrt is not always correctly rounded and its CUDA sqrt is.  At t = 701 of the
    20-step plan the exact sqrt(a_prev) lies 0.5025 ulp above the lower fp32 neighbour; the CPU returns the lower one and
    the GPU the correctly rounded upper one."""
    x, ec = x.to(dtype), ec.to(dtype)
    cast = lambda t: None if t is None else t.to(dtype)
    guide = lambda c, u: c if u is None else u + scale * (c - u)
    e = guide(ec, cast(eu))
    if en is not None:
        ep = (e + guide(cast(en[0]), cast(en[1]))) / 2
    else:
        o = [cast(t) for t in old]
        ep = [lambda: e, lambda: (3 * e - o[0]) / 2, lambda: (23 * e - 16 * o[0] + 5 * o[1]) / 12,
              lambda: (55 * e - 59 * o[0] + 37 * o[1] - 9 * o[2]) / 24][len(old)]()
    full = lambda v: torch.full((x.shape[0], 1, 1, 1), v, device=x.device, dtype=dtype)
    s1m = full(st.sqrt_one_minus_at)
    if dtype == torch.float32:
        sqrt_a_t, sqrt_a_prev, dir_coef = full(st.sqrt_a_t), full(st.sqrt_a_prev), full(st.dir_coef)
    else:
        a_t, a_prev, sigma_t = full(st.a_t), full(st.a_prev), full(st.sigma_t)
        sqrt_a_t, sqrt_a_prev, dir_coef = a_t.sqrt(), a_prev.sqrt(), (1. - a_prev - sigma_t ** 2).sqrt()
    pred_x0 = (x - s1m * ep) / sqrt_a_t
    x_prev = sqrt_a_prev * pred_x0 + dir_coef * ep
    return x_prev, pred_x0, e


@pytest.mark.parametrize("order", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("guided", [False, True])
def test_plms_update_kernel(g, order, guided):
    """Every step of a 20-step SD1.5 plan at SD1.5 latent size: x_prev, pred_x0 and the history slot equal the torch
    fp32 expression bit for bit and stay within F64_TOL of fp64; no input is written."""
    from ctrlora_b200 import ops, plms_schedule
    ref = g["schedule"][20]
    steps = plms_schedule.time_range(ref["ddim_timesteps"])
    plan = plms_schedule.plan(steps, ref["ddim_alphas"], ref["ddim_alphas_prev"], ref["ddim_sqrt_one_minus_alphas"],
                              ref["ddim_sigmas"])
    gen = torch.Generator(device="cuda").manual_seed(100 + 10 * order + guided)
    shape, scale = (4, 4, 64, 64), 7.5
    mk = lambda: torch.randn(shape, device="cuda", generator=gen)
    worst = 0.0
    for st in plan:
        x, ec = mk(), mk()
        eu = mk() if guided else None
        en = (mk(), mk() if guided else None) if order == 0 else None
        old = [mk() for _ in range(max(order - 1, 0))]
        inputs = [t for t in [x, ec, eu, *(en or ()), *old] if t is not None]
        before = [t.clone() for t in inputs]
        e_out = torch.full(shape, float("nan"), device="cuda")
        kw = dict(e_next=en) if order == 0 else dict(old=old)
        x_prev, pred_x0 = ops.plms_update(x, ec, eu, e_out, scale, **st.kernel_args(), **kw)
        rx, rp, re = _torch_update(x, ec, eu, en, old, scale, st, torch.float32)
        assert torch.equal(x_prev, rx) and torch.equal(pred_x0, rp), f"order {order}, step t={st.t}"
        assert torch.equal(e_out, re), "history slot"
        assert all(torch.equal(a, b) for a, b in zip(inputs, before)), "an input was written"
        dx, dp, _ = _torch_update(x, ec, eu, en, old, scale, st, torch.float64)
        worst = max(worst, ((x_prev.double() - dx).norm() / dx.norm()).item(),
                    ((pred_x0.double() - dp).norm() / dp.norm()).item())
    print(f"plms update order {order} guided={guided}: bit-exact to fp32 torch; vs fp64 worst norm-relative {worst:.2e}")
    assert worst < F64_TOL


def test_plms_update_rejects_inputs_the_order_does_not_read():
    from ctrlora_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(2, 4, 8, 8, device="cuda")
    p, n = x.data_ptr(), x.numel()
    args = lambda en, o1, o2, o3, order: (p, p, None, en, None, o1, o2, o3, p, p, p, order, n, 1.0, 1.0, 0.5, 1.0, 0.5,
                                         None)
    assert lib.ctrlora_plms_update(*args(None, p, None, None, 2)) == 0
    torch.cuda.synchronize()
    for bad in (args(None, None, None, None, 2), args(None, p, p, None, 2), args(p, p, None, None, 0),
                args(None, None, None, None, 0), args(p, None, None, None, 1), args(None, p, p, p, 5)):
        assert lib.ctrlora_plms_update(*bad) == 1


# ------------------------------------------------------------------------------------------------ samples vs reference
@pytest.mark.parametrize("steps", [1, 4, 20])
@pytest.mark.parametrize("scale", [1.0, 7.5])
def test_finetune_samples_vs_reference(g, tiny, steps, scale):
    d = tiny_inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]} if scale != 1.0 else None
    outs = _all_policies(tiny, steps, cond, ucond, scale, d["x_T"], g["finetune"][(steps, scale)],
                         BOUND["tiny_finetune"], f"tiny finetune PLMS steps {steps} scale {scale}", graphed=True)
    if scale != 1.0:
        e = rel(outs[(True, True)], outs[(False, True)])
        print(f"  batched vs sequential CFG: rel {e:.2e}")
        assert e < BOUND["cfg_policy"]


def test_intermediates_vs_reference(g, tiny):
    d = tiny_inputs(g)
    ref = g["finetune_intermediates"]
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]}
    with torch.no_grad():
        out, inter, _ = _sample(tiny, ref["steps"], cond, ucond, 7.5, d["x_T"], log_every_t=ref["log_every_t"])
    assert len(inter["x_inter"]) == len(ref["x_inter"]) and len(inter["pred_x0"]) == len(ref["pred_x0"])
    assert inter["x_inter"][0] is d["x_T"] and inter["pred_x0"][0] is d["x_T"] and inter["x_inter"][-1] is out
    err = max(max(rel(a, b) for a, b in zip(inter[k][1:], ref[k][1:])) for k in ("x_inter", "pred_x0"))
    print(f"tiny finetune PLMS intermediates: worst rel err {err:.2e}")
    assert err < BOUND["tiny_intermediates"]


@pytest.mark.parametrize("task", ["canny", "depth", "seg"])
def test_pretrain_samples_vs_reference(g, variants, task):
    model = build(os.path.join(GOLD, "tiny_pretrain.yaml"), variants["pretrain_control_shapes"], variants["unet_shapes"],
                  variants["seed"])
    d = tiny_inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]], "task": task}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]], "task": task}
    # the `task` string keeps the pretrain conditioning off the graph path: eager under every policy
    _all_policies(model, 4, cond, ucond, 7.5, d["x_T"], g["pretrain"][task], BOUND["tiny_pretrain"],
                  f"tiny pretrain ({task}) PLMS steps 4 scale 7.5", graphed=False)


def _inference_model(g, variants):
    model = build(os.path.join(GOLD, "tiny_inference.yaml"), variants["inference_control_shapes"],
                  variants["unet_shapes"], variants["seed"])
    model.lora_weights = list(g["inference_lora_weights"])
    d = tiny_inputs(g)
    conds = [{"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}, {"c_crossattn": [d["ctx"]], "c_concat": [d["hint2"]]}]
    uconds = [{"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]}, {"c_crossattn": [d["uc"]], "c_concat": [d["hint2"]]}]
    return model, d, conds, uconds


def test_inference_two_loras_samples_vs_reference(g, variants):
    model, d, conds, uconds = _inference_model(g, variants)
    # a list of dicts is not on the graph path: every policy runs apply_model eagerly and sequentially
    _all_policies(model, 4, conds, uconds, 7.5, d["x_T"], g["inference"], BOUND["tiny_inference"],
                  "tiny inference (2 LoRAs, weights 0.7 / 0.3) PLMS steps 4 scale 7.5", graphed=False)


def test_style_samples_vs_reference(g):
    st = torch.load(os.path.join(GOLD, "tiny_style_golden.pt"), weights_only=False)
    model = build(os.path.join(GOLD, "tiny_style.yaml"), st["control_shapes"], st["unet_shapes"], st["seed"])
    d = tiny_inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]], "c_ip": [d["ip"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]], "c_ip": [d["uc_ip"]]}
    _all_policies(model, 4, cond, ucond, 7.5, d["x_T"], g["style"], BOUND["tiny_style"],
                  "tiny style (c_ip) PLMS steps 4 scale 7.5", graphed=True)
    # guess mode as the style app sets it: control scales 0.825^(12-i), the uncond without hint.  With c_concat [None]
    # the uncond is off the graph path, so CFG runs sequentially under every policy and only the cond half is replayed
    model.control_scales = list(g["style_guess_control_scales"])
    guess = _all_policies(model, 4, cond, dict(ucond, c_concat=[None]), 7.5, d["x_T"], g["style_guess"],
                          BOUND["tiny_style"], "tiny style guess mode PLMS steps 4 scale 7.5", graphed=True)
    with torch.no_grad():
        app_form = _sample(model, 4, cond, dict(ucond, c_concat=None), 7.5, d["x_T"])[0]   # the app's `None`
    assert torch.equal(app_form, guess[(True, True)])


@pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")
def test_sd15_samples_vs_reference():
    from oracle import synth
    g = torch.load(os.path.join(GOLD, "sd15_plms_golden.pt"), weights_only=False)
    shapes = torch.load(os.path.join(GOLD, "sd15_rank128_golden.pt"), weights_only=False)
    model = build(os.path.join(ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml"), shapes["control_shapes"],
                  shapes["unet_shapes"], g["seed"])
    B, R, seed = g["B"], g["R"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    x_T, hint = mk("plms_xT", (B, 4, R, R)), mk("hint", (B, 4, R, R))
    cond = {"c_crossattn": [mk("ctx", (B, 77, 768))], "c_concat": [hint]}
    ucond = {"c_crossattn": [mk("uc_ctx", (B, 77, 768))], "c_concat": [hint]}
    with torch.no_grad():
        outs = {pol: _sample(model, g["steps"], cond, ucond, g["scale"], x_T, *pol)[0]
                for pol in ((True, True), (True, False), (False, True))}
    e = max(rel(o, g["samples"]) for o in outs.values())
    print(f"SD1.5 rank128 PLMS batch {B} steps {g['steps']} scale {g['scale']}: rel err {e:.2e}")
    assert e < BOUND["sd15"]
    assert torch.equal(outs[(True, True)], outs[(True, False)])
    e = rel(outs[(True, True)], outs[(False, True)])
    print(f"  batched vs sequential CFG: rel {e:.2e}")
    assert e < BOUND["cfg_policy"]


# ------------------------------------------------------------------------------------------------ the loop itself
def _reference_loop(model, calls, x_T, steps, scale, mask, x0):
    """plms_sampling / p_sample_plms (plms.py:128-244) in torch, eta 0, with every apply_model answered from `calls`
    (the sampler's own (x, t, eps) in call order, cond before uncond) after checking that the loop asks at the same x
    and t.  noise_like is not drawn (its product with sigma_t = 0 is zero), so q_sample's draws line up."""
    from ldm.modules.diffusionmodules.util import make_ddim_sampling_parameters, make_ddim_timesteps
    it = iter(calls)

    def model_output(x, t):
        (xc, tc, ec), (xu, tu, eu) = next(it), next(it)
        assert torch.equal(xc, x) and torch.equal(tc, t) and torch.equal(xu, x) and torch.equal(tu, t)
        return eu + scale * (ec - eu)
    timesteps = make_ddim_timesteps("uniform", steps, 1000, verbose=False)
    sigmas, alphas, alphas_prev = make_ddim_sampling_parameters(model.alphas_cumprod.cpu(), timesteps, 0., verbose=False)
    s1m = np.sqrt(1. - alphas)
    b, dev = x_T.shape[0], x_T.device
    time_range = np.flip(timesteps)
    img, old_eps, out = x_T, [], {"x": [], "pred_x0": []}
    for i, step in enumerate(time_range):
        index = len(time_range) - i - 1
        ts = torch.full((b,), step, device=dev, dtype=torch.long)
        ts_next = torch.full((b,), time_range[min(i + 1, len(time_range) - 1)], device=dev, dtype=torch.long)
        img_orig = model.q_sample(x0, ts)
        img = img_orig * mask + (1. - mask) * img
        full = lambda v: torch.full((b, 1, 1, 1), v, device=dev)
        a_t, a_prev, sigma_t, sq = full(alphas[index]), full(alphas_prev[index]), full(sigmas[index]), full(s1m[index])

        def x_prev_and_pred_x0(e_t, x=img):
            pred_x0 = (x - sq * e_t) / a_t.sqrt()
            return a_prev.sqrt() * pred_x0 + (1. - a_prev - sigma_t ** 2).sqrt() * e_t, pred_x0
        e_t = model_output(img, ts)
        if not old_eps:
            e_t_prime = (e_t + model_output(x_prev_and_pred_x0(e_t)[0], ts_next)) / 2
        elif len(old_eps) == 1:
            e_t_prime = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:
            e_t_prime = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:
            e_t_prime = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        img, pred_x0 = x_prev_and_pred_x0(e_t_prime)
        old_eps = (old_eps + [e_t])[-3:]
        out["x"].append(img)
        out["pred_x0"].append(pred_x0)
    assert next(it, None) is None
    return out


def test_loop_with_mask_and_callbacks_follows_the_reference(g, tiny):
    """Sequential CFG, eager: every model input, history entry, x0 / mask blend (q_sample's noise from the same seed),
    pred_x0 handed to img_callback and x_prev kept in the intermediates equals the reference loop's, bit for bit;
    callback(i) and img_callback(pred_x0, i) come once per step in order."""
    d = tiny_inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]}
    x0 = d["hint"].flip(0).contiguous()
    mask = torch.zeros(d["x_T"].shape[0], 1, 16, 16, device="cuda")
    mask[..., 8:] = 1.
    calls, cbs, imgs = [], [], []
    real = tiny.apply_model

    def recording(x, t, c):
        e = real(x, t, c)
        calls.append((x.clone(), t.clone(), e.float().clone()))
        return e
    tiny.apply_model = recording
    try:
        torch.manual_seed(1234)
        with torch.no_grad():
            out, inter, _ = _sample(tiny, 5, cond, ucond, 7.5, d["x_T"], batched_cfg=False, use_cuda_graph=False,
                                 mask=mask, x0=x0, log_every_t=1, callback=cbs.append,
                                 img_callback=lambda p, i: imgs.append((p.clone(), i)))
    finally:
        del tiny.apply_model
    assert len(calls) == 2 * (5 + 1)
    torch.manual_seed(1234)
    with torch.no_grad():
        ref = _reference_loop(tiny, calls, d["x_T"], 5, 7.5, mask, x0)
    assert cbs == list(range(5)) and [i for _, i in imgs] == list(range(5))
    assert all(torch.equal(p, r) for (p, _), r in zip(imgs, ref["pred_x0"]))
    assert all(torch.equal(a, b) for a, b in zip(inter["x_inter"][1:], ref["x"]))
    assert all(torch.equal(a, b) for a, b in zip(inter["pred_x0"][1:], ref["pred_x0"]))
    assert torch.equal(out, ref["x"][-1])


def test_one_sampler_recaptures_across_a_lora_switch(g):
    """The gradio apps keep one sampler across LoRA changes.  On the finetune model with dict conditioning (the graph
    path, batched CFG), LoRA factors reloaded in place make the reused sampler's private DDIMSampler capture a new graph
    under a new key, and its samples equal a fresh sampler's and an eager run's."""
    from ldm.models.diffusion.plms import PLMSSampler
    from oracle import synth
    shapes = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = build(os.path.join(GOLD, "tiny_finetune.yaml"), shapes["control_shapes"], shapes["unet_shapes"],
                  shapes["seed"])   # its own model: the test rewrites its weights
    d = tiny_inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]}
    run = lambda s: s.sample(4, d["x_T"].shape[0], (4, 16, 16), cond, verbose=False, x_T=d["x_T"],
                             unconditional_guidance_scale=7.5, unconditional_conditioning=ucond)[0].clone()
    lora = {k: v for k, v in shapes["control_shapes"].items() if "lora_layer" in k}
    assert lora
    with torch.no_grad():
        reused = PLMSSampler(model)
        first = run(reused)
        graph, key = reused.eps_model._graph, reused.eps_model._graph_key
        assert graph is not None
        model.control_model.load_state_dict(synth.synth_state_dict(lora, shapes["seed"] + 1, "control_model."),
                                            strict=False)
        switched = run(reused)
        assert reused.eps_model._graph is not graph and reused.eps_model._graph_key != key
        assert torch.equal(switched, run(PLMSSampler(model)))
        assert torch.equal(switched, run(PLMSSampler(model, use_cuda_graph=False)))
    assert rel(first, switched) > 1e-3
