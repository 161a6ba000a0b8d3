"""Parity of the API surfaces round 1 left untested, against outputs of the UNMODIFIED reference
(tests/golden/tiny_variants_golden.pt, produced by `tools/make_golden.py --variants`):

  * ControlPretrainLDM.apply_model per task                  cldm/cldm_ctrlora_pretrain.py:95-111
  * ControlInferenceLDM.apply_model, 2 LoRA sets + weights    cldm/cldm_ctrlora_inference.py:156-178
  * DDIMSampler.encode / decode / stochastic_encode           cldm/ddim_hacked.py:233-317
  * finetune training step with only_mid_control=True         cldm/cldm.py:39-42

Metric: norm-relative error.  Tolerances: north_star asks 1e-3 relative fp16; the measured figure for this tiny,
random-init network is printed and the assert sits at TOL (see tests/tolerances.py for how each bound was set).
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu

from tolerances import TOL  # noqa: E402
from golden_io import load_golden  # noqa: E402


def rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / (ref.norm() + 1e-20)).item()


@pytest.fixture(scope="module")
def g():
    return load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))


def build(kind, g, control_shapes):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from oracle import synth
    model = create_model(os.path.join(GOLD, f"tiny_{kind}.yaml"), init_weights=False)
    model.control_model.load_state_dict(synth.synth_state_dict(control_shapes, g["seed"], "control_model."), strict=True)
    model.model.diffusion_model.load_state_dict(
        synth.synth_state_dict(g["unet_shapes"], g["seed"], "model.diffusion_model."), strict=True)
    return model.cuda().eval()


def inputs(g):
    from oracle import synth
    B, H, seed = g["B"], g["H"], g["seed"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    return dict(x=mk("x", (B, 4, H, H)), hint=mk("hint", (B, 4, H, H)), hint2=mk("hint2", (B, 4, H, H)),
                ctx=mk("ctx", (B, 77, 64)), uc=mk("uc_ctx", (B, 77, 64)), noise=mk("noise", (B, 4, H, H)), t=g["t"].cuda())


def test_pretrain_apply_model_vs_reference(g):
    model = build("pretrain", g, g["pretrain_control_shapes"])
    assert list(model.control_model.state_dict().keys()) == g["pretrain_key_order"]
    d = inputs(g)
    errs = {}
    with torch.no_grad():
        for task in ("canny", "depth", "seg", "canny"):
            eps = model.apply_model(d["x"], d["t"], {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]], "task": task})
            errs[task] = rel(eps, g[f"pretrain_eps_{task}"])
        eps = model.apply_model(d["x"], d["t"], {"c_crossattn": [d["ctx"]], "c_concat": None, "task": "canny"})
        errs["nocontrol"] = rel(eps, g["pretrain_eps_nocontrol"])
    print("pretrain apply_model rel errors:", {k: "%.2e" % v for k, v in errs.items()})
    assert max(errs.values()) < TOL["tiny_eps"]
    assert rel(g["pretrain_eps_canny"], g["pretrain_eps_depth"]) > 1e-2  # the task's LoRA set matters


def test_inference_apply_model_weighted_sum_vs_reference(g):
    model = build("inference", g, g["inference_control_shapes"])
    assert list(model.control_model.state_dict().keys()) == g["inference_key_order"]
    d = inputs(g)
    conds = [{"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}, {"c_crossattn": [d["ctx"]], "c_concat": [d["hint2"]]}]
    with torch.no_grad():
        e_def = rel(model.apply_model(d["x"], d["t"], conds), g["inference_eps_default"])
        model.lora_weights = [0.7, 0.3]
        model.control_scales = [0.5 + 0.1 * i for i in range(13)]
        eps_grouped = model.apply_model(d["x"], d["t"], conds)   # default: both LoRA sets in ONE ControlNet pass
        e_w = rel(eps_grouped, g["inference_eps_weighted"])
        model.grouped_multi_lora = False                          # the reference's loop: one ControlNet pass per set
        eps_seq = model.apply_model(d["x"], d["t"], conds)
        model.grouped_multi_lora = True
        assert torch.equal(eps_grouped, eps_seq), rel(eps_grouped, eps_seq)  # same kernels per image: bit-identical
        model.control_scales = [1.0] * 13
        cerr = []
        for i in (0, 1):
            model.control_model.switch_lora(i)
            got = model.control_model(hint=d["hint"], timesteps=d["t"], context=d["ctx"])
            cerr.append(max(rel(a, b) for a, b in zip(got, g[f"inference_control_{i}"])))
    print(f"inference apply_model: default weights {e_def:.2e}, weighted+scaled {e_w:.2e}, control stacks {cerr}")
    assert max(e_def, e_w) < TOL["tiny_eps"] and max(cerr) < TOL["tiny_control"]
    assert rel(g["inference_eps_default"], g["inference_eps_weighted"]) > 1e-2  # the weights / scales matter
    with pytest.raises(AssertionError):  # reference :159-161
        model.apply_model(d["x"], d["t"], conds[:1] * 3)


def test_sampler_encode_decode_vs_reference(g):
    from cldm.ddim_hacked import DDIMSampler
    gt = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = build("finetune", g, gt["control_shapes"])
    d = inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]}
    for graph in (False, True):
        s = DDIMSampler(model, use_cuda_graph=graph)
        s.make_schedule(10, ddim_eta=0.0, verbose=False)
        x_enc, out = s.encode(d["x"], cond, 4, return_intermediates=2)
        e_enc = rel(x_enc, g["encode"]["x_encoded"])
        assert out["intermediate_steps"] == g["encode"]["intermediate_steps"]
        assert len(out["intermediates"]) == g["encode"]["n_intermediates"]
        e_dec = rel(s.decode(d["x"], cond, 4, unconditional_guidance_scale=3.0, unconditional_conditioning=ucond), g["decode"])
        st = s.stochastic_encode(d["x"], g["stochastic_encode"]["t"].cuda(), use_original_steps=True, noise=d["noise"])
        # CFG inversion (an extension: the reference's CFG branch cannot run with dict conds) == two eager passes + combine
        if not graph:
            x_cfg, _ = s.encode(d["x"], cond, 2, unconditional_guidance_scale=3.0, unconditional_conditioning=ucond)
            assert torch.isfinite(x_cfg).all() and rel(x_cfg, x_enc) > 1e-4
        print(f"graph={graph}: encode {e_enc:.2e}, decode {e_dec:.2e}")
        assert e_enc < TOL["tiny_sample"] and e_dec < TOL["tiny_sample"]
        assert torch.equal(st.cpu(), g["stochastic_encode"]["out"])  # gather + 2 fp32 products: bit-exact


def test_training_only_mid_control_vs_reference(g):
    from ctrlora_b200.train import FinetuneTrainer
    gt = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = build("finetune", g, gt["control_shapes"])
    model.only_mid_control = True
    d = inputs(g)
    tr = FinetuneTrainer(model, lr=1e-3)
    loss = tr.loss_and_grads(d["x"], d["hint"], d["ctx"], d["t"], d["noise"])
    ref = g["midonly_train"]
    e_loss = abs(loss.item() - ref["loss"].item()) / abs(ref["loss"].item())
    e_eps = rel(tr.last_eps, ref["eps"])
    grads = tr.unscaled_grads()
    norms = sorted(v for v in ref["grad_norms"].values())
    biggest, median = norms[-1], norms[len(norms) // 2]
    worst, n_zero = 0.0, 0
    for n, rn in ref["grad_norms"].items():
        got = grads[n].norm().item()
        if rn < 1e-5 * biggest:  # unused parameter (the 12 skip zero-convs) or exactly-cancelled gradient
            assert got < 1e-2 * median, (n, got, rn)
            n_zero += 1
        else:
            worst = max(worst, abs(got - rn) / rn)
    print(f"only_mid training: loss err {e_loss:.2e}, eps err {e_eps:.2e}, worst grad-norm err {worst:.2e}, {n_zero} zero grads")
    assert e_loss < TOL["tiny_loss"] and e_eps < TOL["tiny_eps"] and worst < TOL["tiny_grad_norm"]
    assert n_zero >= 24  # 12 skip zero-convs x (weight, bias)


def test_graph_follows_load_state_dict(g):
    """ADVICE r1: the sampler's captured graph must not replay stale folded weights after load_state_dict on the SAME
    model (app/gradio_ctrlora.py re-uses one sampler across checkpoints)."""
    from cldm.ddim_hacked import DDIMSampler
    from oracle import synth
    gt = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = build("finetune", g, gt["control_shapes"])
    d = inputs(g)
    cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
    ucond = {"c_crossattn": [d["uc"]], "c_concat": [d["hint"]]}
    B = g["B"]
    ts = torch.full((B,), 981, dtype=torch.long, device="cuda")
    s = DDIMSampler(model, use_cuda_graph=True)
    s.make_schedule(50, ddim_eta=0.0, verbose=False)
    kw = dict(index=49, unconditional_guidance_scale=7.5, unconditional_conditioning=ucond)
    x1, _ = s.p_sample_ddim(d["x"], cond, ts, **kw)
    x1 = x1.clone()
    new_sd = synth.synth_state_dict(gt["control_shapes"], g["seed"] + 1, "control_model.")
    model.control_model.load_state_dict(new_sd, strict=True)
    x2, _ = s.p_sample_ddim(d["x"], cond, ts, **kw)          # same sampler, same shapes: graph must be rebuilt
    eager = DDIMSampler(model, use_cuda_graph=False)
    eager.make_schedule(50, ddim_eta=0.0, verbose=False)
    x3, _ = eager.p_sample_ddim(d["x"], cond, ts, **kw)
    # stale folded weights would leave x2 near x1 (the two checkpoints differ by ~0.2); run-to-run noise of the tiny network
    # is ~1e-3 (tools/debug_determinism.py)
    assert rel(x2, x3) < 5e-3, "graph replayed stale weights"
    assert rel(x2, x1) > 5e-2


def test_context_cache_follows_prompt_changes(g):
    """The sampler registers the text context as step-invariant (K / V^T projected once per run): a new prompt through the SAME
    sampler / graph, and in-place edits of the context tensor, must be seen; a call that bypasses the sampler must not hit a
    stale cache."""
    from cldm.ddim_hacked import DDIMSampler
    from oracle import synth
    gt = torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)
    model = build("finetune", g, gt["control_shapes"])
    d = inputs(g)
    B = g["B"]
    ts = torch.full((B,), 981, dtype=torch.long, device="cuda")
    ctx2 = synth.synth_input("ctx_other", (B, 77, 64), g["seed"]).cuda()
    s = DDIMSampler(model, use_cuda_graph=True)
    s.make_schedule(50, ddim_eta=0.0, verbose=False)
    eager = DDIMSampler(model, use_cuda_graph=False, batched_cfg=False)
    eager.make_schedule(50, ddim_eta=0.0, verbose=False)

    def run(smp, ctx, uc):
        cond = {"c_crossattn": [ctx], "c_concat": [d["hint"]]}
        ucond = {"c_crossattn": [uc], "c_concat": [d["hint"]]}
        with smp.run_mode():  # what sample() does: conditioning constant over the run -> context K / V^T cached
            out = smp.p_sample_ddim(d["x"], cond, ts, index=49, unconditional_guidance_scale=7.5, unconditional_conditioning=ucond)[0]
            out2 = smp.p_sample_ddim(d["x"], cond, ts, index=49, unconditional_guidance_scale=7.5, unconditional_conditioning=ucond)[0]
        assert torch.equal(out, out2)  # second step of the run: cache hit, bit-identical (the forward is deterministic)
        return out.clone()

    a1 = run(s, d["ctx"], d["uc"])
    a2 = run(s, ctx2, d["uc"])              # new prompt, same sampler and graph
    ctx3 = d["ctx"].clone()
    a3 = run(s, ctx3, d["uc"])
    ctx3.mul_(0.5)                          # in-place edit of a registered context
    a4 = run(s, ctx3, d["uc"])
    for got, ctx in ((a1, d["ctx"]), (a2, ctx2), (a3, d["ctx"]), (a4, d["ctx"] * 0.5)):
        ref = run(eager, ctx.clone(), d["uc"].clone())
        assert rel(got, ref) < 1e-5, rel(got, ref)
    assert rel(a2, a1) > 1e-3 and rel(a4, a3) > 1e-3
