"""DPM-Solver++ on the sm_90a kernels: the fp32-t time embedding, apply_model at a fractional time, and
DPMSolverSampler.sample against the unmodified reference's DPMSolverSampler (tests/golden/tiny_dpm_golden.pt,
sd15_dpm_golden.pt) under every batched-CFG / CUDA-graph policy.

Bounds follow tests/tolerances.py: the error measured on an H100 when the bound was set, plus 20 %, written beside it."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pytestmark = pytest.mark.gpu

from golden_io import load_golden  # noqa: E402
from tolerances import TOL  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
EMB_ABS = 4 * 2.0 ** -23   # fractional-t embedding vs torch fp32 cos / sin of the same product: 4 ulp of 1.0 (measured 0)
BOUND = {                  # norm-relative error of the final sample vs the reference's (H100, measured)
    "tiny_finetune": 4.3e-3,   # 3.60e-3 worst of steps 4 / 5 / 16 with and without CFG (steps 4, CFG 7.5)
    "tiny_inference": 4.7e-3,  # 3.89e-3 (2 LoRAs, steps 5, CFG 7.5)
    "sd15": 4.2e-3,            # 3.47e-3 (SD1.5 rank 128, steps 3, CFG 7.5)
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
    return torch.load(os.path.join(GOLD, "tiny_dpm_golden.pt"), weights_only=False)


@pytest.fixture(scope="module")
def shapes():
    return torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)


@pytest.fixture(scope="module")
def tiny(shapes):
    return build(os.path.join(GOLD, "tiny_finetune.yaml"), shapes["control_shapes"], shapes["unet_shapes"], shapes["seed"])


def tiny_inputs(g):
    from oracle import synth
    B, H, seed = g["B"], g["H"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    return (mk("dpm_xT", (B, 4, H, H)), mk("hint", (B, 4, H, H)), mk("hint2", (B, 4, H, H)), mk("ctx", (B, 77, 64)),
            mk("uc_ctx", (B, 77, 64)))


def test_f32_embedding_integer_t_matches_int64_bits():
    from ctrlora_b200 import dropin
    dropin.activate()
    from ldm.modules.diffusionmodules.util import timestep_embedding
    t = torch.tensor([0, 1, 21, 500, 949, 981, 999], device="cuda")
    for dim in (32, 320):
        assert torch.equal(timestep_embedding(t.float(), dim), timestep_embedding(t, dim))


def test_f32_embedding_fractional_t_vs_torch(g):
    from ctrlora_b200 import dropin
    dropin.activate()
    from ldm.modules.diffusionmodules.util import embedding_freqs, timestep_embedding
    t = torch.tensor(g["schedule"][20]["model_time"] + [0.5, 123.456], dtype=torch.float32, device="cuda")
    got = timestep_embedding(t, 320)
    arg = t[:, None] * embedding_freqs(320, 10000, t.device)[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], -1)
    err = (got - ref).abs().max().item()
    print(f"fp32-t embedding: max abs err {err:.3e} vs torch cos/sin (bound {EMB_ABS:.3e})")
    assert err <= EMB_ABS
    # the int64 path would have truncated these: 949.05 and 949 embed differently
    assert not torch.equal(got, timestep_embedding(t.long(), 320))


def test_apply_model_at_fractional_t_vs_oracle(tiny, shapes):
    from oracle import ctrlora_oracle as O
    from oracle import synth
    seed = shapes["seed"]
    x, hint = synth.synth_input("x", (2, 4, 16, 16), seed), synth.synth_input("hint", (2, 4, 16, 16), seed)
    ctx = synth.synth_input("ctx", (2, 77, 64), seed)
    t = torch.tensor([949.05, 21.3], dtype=torch.float32)
    sd = {k: v.detach().float().cpu() for k, v in tiny.state_dict().items()}
    with torch.no_grad():
        got = tiny.apply_model(x.cuda(), t.cuda(), {"c_crossattn": [ctx.cuda()], "c_concat": [hint.cuda()]})
        ref = O.apply_model(sd, x, t, ctx, hint, 4, 32)
    e = rel(got, ref)
    print(f"apply_model at t = {t.tolist()}: rel err {e:.2e} vs the CPU oracle")
    assert e < TOL["tiny_eps"]


def _sample(model, steps, cond, ucond, scale, x_T, batched_cfg, use_cuda_graph):
    from ldm.models.diffusion.dpm_solver.sampler import DPMSolverSampler
    sampler = DPMSolverSampler(model, batched_cfg=batched_cfg, use_cuda_graph=use_cuda_graph)
    out, none = sampler.sample(steps, x_T.shape[0], tuple(x_T.shape[1:]), cond, verbose=False, x_T=x_T,
                               unconditional_guidance_scale=scale, unconditional_conditioning=ucond)
    assert none is None and out.dtype == torch.float32 and out.device == x_T.device
    return out


@pytest.mark.parametrize("steps", [4, 5, 16])
@pytest.mark.parametrize("scale", [1.0, 7.5])
def test_finetune_samples_vs_reference(g, tiny, steps, scale):
    x_T, hint, _, ctx, uc = tiny_inputs(g)
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    ref = g["finetune"][(steps, scale)]
    outs = {}
    with torch.no_grad():
        for pol in POLICIES:
            outs[pol] = _sample(tiny, steps, cond, ucond if scale != 1.0 else None, scale, x_T, *pol)
    errs = {pol: rel(o, ref) for pol, o in outs.items()}
    print(f"tiny finetune DPM++ steps {steps} scale {scale}: rel err {max(errs.values()):.2e}")
    assert max(errs.values()) < BOUND["tiny_finetune"]
    for batched in (True, False):
        assert torch.equal(outs[(batched, True)], outs[(batched, False)])  # graph replay == eager, bit for bit


def test_inference_two_loras_samples_vs_reference(g):
    shapes = load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))
    model = build(os.path.join(GOLD, "tiny_inference.yaml"), shapes["inference_control_shapes"], shapes["unet_shapes"],
                  shapes["seed"])
    model.lora_weights = list(g["inference_lora_weights"])
    x_T, hint, hint2, ctx, uc = tiny_inputs(g)
    conds = [{"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [ctx], "c_concat": [hint2]}]
    uconds = [{"c_crossattn": [uc], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint2]}]
    ref = g["inference"][(5, 7.5)]
    with torch.no_grad():
        outs = {pol: _sample(model, 5, conds, uconds, 7.5, x_T, *pol) for pol in POLICIES}
    e = max(rel(o, ref) for o in outs.values())
    print(f"tiny inference (2 LoRAs) DPM++ steps 5 scale 7.5: rel err {e:.2e}")
    assert e < BOUND["tiny_inference"]
    for batched in (True, False):
        assert torch.equal(outs[(batched, True)], outs[(batched, False)])


@pytest.mark.skipif(os.environ.get("CTRLORA_SKIP_FULL") == "1", reason="CTRLORA_SKIP_FULL=1")
def test_sd15_samples_vs_reference():
    from oracle import synth
    g = torch.load(os.path.join(GOLD, "sd15_dpm_golden.pt"), weights_only=False)
    shapes = torch.load(os.path.join(GOLD, "sd15_rank128_golden.pt"), weights_only=False)
    model = build(os.path.join(ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml"), shapes["control_shapes"],
                  shapes["unet_shapes"], g["seed"])
    B, R, seed = g["B"], g["R"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    x_T, hint = mk("dpm_xT", (B, 4, R, R)), mk("hint", (B, 4, R, R))
    cond, ucond = {"c_crossattn": [mk("ctx", (B, 77, 768))], "c_concat": [hint]}, \
        {"c_crossattn": [mk("uc_ctx", (B, 77, 768))], "c_concat": [hint]}
    with torch.no_grad():
        outs = {pol: _sample(model, g["steps"], cond, ucond, g["scale"], x_T, *pol) for pol in ((True, True), (True, False))}
    e = max(rel(o, g["samples"]) for o in outs.values())
    print(f"SD1.5 rank128 DPM++ steps {g['steps']} scale {g['scale']}: rel err {e:.2e}")
    assert e < BOUND["sd15"]
    assert torch.equal(outs[(True, True)], outs[(True, False)])


def test_ddim_unchanged_by_float_t_on_the_same_sampler(g, tiny):
    """One DDIMSampler serves int64 t (its own steps) and float t (what DPM-Solver feeds it): its graphs and CFG
    buffers are keyed on t's dtype, so DDIM sampling is bit-identical before and after, and the float-t eps equals an
    eager apply_model at the untruncated time."""
    from cldm.ddim_hacked import DDIMSampler
    x_T, hint, _, ctx, uc = tiny_inputs(g)
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    ddim = DDIMSampler(tiny, batched_cfg=True, use_cuda_graph=True)
    run = lambda: ddim.sample(4, x_T.shape[0], (4, 16, 16), cond, verbose=False, x_T=x_T, unconditional_guidance_scale=7.5,
                              unconditional_conditioning=ucond)[0].clone()
    with torch.no_grad():
        before = run()
        t = torch.full((x_T.shape[0],), 949.05, device="cuda")
        e_c, e_u = (e.clone() for e in ddim._eps_pair(x_T, t, cond, ucond, True))   # batched CFG, graph replay
        _sample(tiny, 5, cond, ucond, 7.5, x_T, True, True)   # a DPM run on the same model in between
        after = run()
        both = {"c_crossattn": [torch.cat([ctx, uc])], "c_concat": [torch.cat([hint, hint])]}
        ref = tiny.apply_model(torch.cat([x_T, x_T]), torch.cat([t, t]), both)
        trunc = tiny.apply_model(torch.cat([x_T, x_T]), torch.cat([t, t]).long(), both)
    b = x_T.shape[0]
    assert torch.equal(before, after)
    assert torch.equal(e_c, ref[:b]) and torch.equal(e_u, ref[b:])
    assert not torch.equal(e_c, trunc[:b])


@pytest.mark.parametrize("kind", ["pretrain", "inference"])
@pytest.mark.parametrize("scale", [1.0, 7.5])
def test_every_variant_samples(g, kind, scale):
    """the reference's DPMSolverSampler fails on all of these; the drop-in samples them (the finetune model is covered
    against the reference above): finite samples, graph replay == eager"""
    shapes = load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))
    model = build(os.path.join(GOLD, f"tiny_{kind}.yaml"), shapes[f"{kind}_control_shapes"], shapes["unet_shapes"],
                  shapes["seed"])
    x_T, hint, hint2, ctx, uc = tiny_inputs(g)
    if kind == "pretrain":
        cond = {"c_crossattn": [ctx], "c_concat": [hint], "task": "depth"}
        ucond = {"c_crossattn": [uc], "c_concat": [hint], "task": "depth"}
    else:
        cond = [{"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [ctx], "c_concat": [hint2]}]
        ucond = [{"c_crossattn": [uc], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint2]}]
    with torch.no_grad():
        outs = [_sample(model, 5, cond, ucond if scale != 1.0 else None, scale, x_T, True, graph) for graph in (True, False)]
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
    assert rel(outs[0], x_T) > 1e-2
