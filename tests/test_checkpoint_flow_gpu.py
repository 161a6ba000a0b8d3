"""Checkpoint tooling parity (SURVEY.md §8 row f4): the reference's weight-surgery scripts are pure state-dict key logic
(scripts/tool_extract_weights.py:22-41 `extract_lora` / `extract_control`, scripts/tool_combine_weights.py:20-45, and the load
order of api.py:31-62).  Their filters are restated here verbatim-in-behaviour and run against the DROP-IN modules: a
pretrained base ControlNet's per-task LoRA checkpoints are extracted, loaded into the multi-LoRA inference model in the
api.py order (switch_lora(i) -> load_state_dict(strict=False) -> copy_weights_to_switchable()), and must reproduce the
pretrain model's control stacks; the `_fuse_lora` deployment export must not change the outputs either."""
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


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def extract_lora(ckpt):      # scripts/tool_extract_weights.py:22-33
    out = {}
    for k in ckpt.keys():
        if 'control_model' in k and 'loras_dict' not in k:
            if 'lora_layer' in k or 'zero_convs' in k or 'middle_block_out' in k or 'norm' in k:
                out[k] = ckpt[k]
    return out


def extract_control(ckpt):   # scripts/tool_extract_weights.py:36-41
    return {k: v for k, v in ckpt.items() if 'control_model' in k and 'loras_dict' not in k}


def check_key(k):            # api.py:27-29
    return 'lora_layer' in k or 'zero_convs' in k or 'middle_block_out' in k or 'norm' in k


def test_extract_combine_load_flow_reproduces_the_pretrained_tasks():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.cldm_ctrlora_pretrain import ControlPretrainLDM
    from cldm.lora import LoRACompatibleLinear
    from cldm.model import create_model
    from oracle import synth
    g = load_golden(os.path.join(GOLD, "tiny_variants_golden.pt"))
    seed = g["seed"]
    pre = create_model(os.path.join(GOLD, "tiny_pretrain.yaml"), init_weights=False)
    assert isinstance(pre, ControlPretrainLDM)
    pre.control_model.load_state_dict(synth.synth_state_dict(g["pretrain_control_shapes"], seed, "control_model."))
    pre.model.diffusion_model.load_state_dict(synth.synth_state_dict(g["unet_shapes"], seed, "model.diffusion_model."))
    pre = pre.cuda().eval()
    # --- tool_extract_weights.py --type lora --from_base: one checkpoint per task (:56-66)
    pre.control_model.switch_lora('canny')
    task_ckpts = {}
    for task in pre.control_model.tasks:
        pre.control_model.switch_lora(task)
        task_ckpts[task] = {k: v.detach().cpu().clone() for k, v in extract_lora(pre.state_dict()).items()}
        assert any('lora_layer.down.weight' in k for k in task_ckpts[task])
    # --- tool_extract_weights.py --type control, tool_combine_weights.py
    base_ckpt = {k: v.detach().cpu().clone() for k, v in extract_control(pre.state_dict()).items()}
    sd_ckpt = {k: v.detach().cpu().clone() for k, v in pre.state_dict().items() if k.startswith("model.diffusion_model.")}
    combined = {}
    combined.update(sd_ckpt); combined.update(base_ckpt); combined.update(task_ckpts['depth']); combined.update({'logvar': torch.zeros(1000)})
    fin = create_model(os.path.join(GOLD, "tiny_finetune.yaml"), init_weights=False)
    missing, unexpected = fin.load_state_dict(combined, strict=False)
    assert not unexpected and all(m.startswith(("first_stage_model.", "cond_stage_model.")) or "posterior" in m or m in (
        "betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod",
        "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod") for m in missing), missing
    fin = fin.cuda().eval()
    # --- api.py:45-62: inference model with two LoRA sets (depth, seg)
    inf = create_model(os.path.join(GOLD, "tiny_inference.yaml"), init_weights=False).cuda().eval()
    inf.load_state_dict(sd_ckpt, strict=False)
    inf.load_state_dict({k: v for k, v in base_ckpt.items() if k.startswith('control_model') and not check_key(k)}, strict=False)
    for i, task in enumerate(('depth', 'seg')):
        inf.control_model.switch_lora(i)
        inf.load_state_dict({k: v for k, v in task_ckpts[task].items() if check_key(k)}, strict=False)
        inf.control_model.copy_weights_to_switchable()
    B, H = g["B"], g["H"]
    mk = lambda n, s: synth.synth_input(n, s, seed).cuda()
    hint, ctx, t = mk("hint", (B, 4, H, H)), mk("ctx", (B, 77, 64)), g["t"].cuda()
    with torch.no_grad():
        want = {}
        for task in ('depth', 'seg'):
            pre.control_model.switch_lora(task)
            want[task] = [c.float().clone() for c in pre.control_model(hint=hint, timesteps=t, context=ctx)]
        errs = []
        for i, task in enumerate(('depth', 'seg')):
            inf.control_model.switch_lora(i)
            got = inf.control_model(hint=hint, timesteps=t, context=ctx)
            errs.append(max(rel(a, b) for a, b in zip(got, want[task])))
        got_fin = fin.control_model(hint=hint, timesteps=t, context=ctx)
        e_fin = max(rel(a, b) for a, b in zip(got_fin, want['depth']))
        # deployment export: fold every LoRA into its linear (cldm/lora.py:237-267), drop the LoRA layers
        for m in fin.control_model.modules():
            if isinstance(m, LoRACompatibleLinear):
                m._fuse_lora()
                assert m.lora_layer is None
        got_fused = fin.control_model(hint=hint, timesteps=t, context=ctx)
        e_fused = max(rel(a, b) for a, b in zip(got_fused, want['depth']))
    print(f"inference sets vs pretrain tasks {errs}, combined finetune ckpt {e_fin:.2e}, after _fuse_lora {e_fused:.2e}")
    # same weights through three different module trees: only run-to-run / fold-order noise is allowed
    assert max(errs + [e_fin, e_fused]) < TOL["tiny_control"]
    assert rel(want['depth'][-1], want['seg'][-1]) > 1e-2
