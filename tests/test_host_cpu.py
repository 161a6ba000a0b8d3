"""CPU-side checks (no GPU, no compute calls into the library): the C ABI loads and exports every declared symbol,
the drop-in module tree reproduces the reference's state-dict keys / shapes / order, the host-side schedule and
sampler tables are bit-exact against the golden fixture, and the product fails loudly without a GPU."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def g():
    return torch.load(os.path.join(GOLD, "tiny_finetune_golden.pt"), weights_only=False)


@pytest.fixture(scope="module")
def tiny_model():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    return create_model(os.path.join(GOLD, "tiny_finetune.yaml"))


def test_abi_exports_every_declared_symbol():
    from ctrlora_b200 import _lib
    header = open(os.path.join(ROOT, "include", "ctrlora_b200.h")).read()
    declared = set(re.findall(r"\b(ctrlora_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    lib = _lib.load()
    for name in declared:
        assert getattr(lib, name) is not None


def test_abi_version_is_3():
    """version 3: ctrlora_groupnorm_args has no stats_prezeroed field, so the struct layout differs from version 2"""
    from ctrlora_b200 import _lib
    assert _lib.load().ctrlora_abi_version() == 3


def test_gemm_args_struct_layout_matches_header():
    """ctypes mirror vs the C struct: same field order (sizes are checked implicitly by the GPU parity tests)."""
    from ctrlora_b200 import _lib
    header = open(os.path.join(ROOT, "include", "ctrlora_b200.h")).read()
    body = header[header.index("typedef struct ctrlora_gemm_args {"):header.index("} ctrlora_gemm_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split("{", 1)[1].split(";"):
        decl = decl.strip()
        if not decl:
            continue
        for part in decl.split(","):
            names.append(re.sub(r"\[.*\]", "", part.strip().split()[-1].lstrip("*")))
    assert names == [f[0] for f in _lib.GemmArgs._fields_]


def test_state_dict_tree_matches_reference(g, tiny_model):
    cn = tiny_model.control_model.state_dict()
    un = tiny_model.model.diffusion_model.state_dict()
    assert list(cn.keys()) == g["control_key_order"]
    assert list(un.keys()) == g["unet_key_order"]
    assert {k: tuple(v.shape) for k, v in cn.items()} == g["control_shapes"]
    assert {k: tuple(v.shape) for k, v in un.items()} == g["unet_shapes"]
    assert len(tiny_model.control_scales) == 13 and not hasattr(tiny_model.control_model, "input_hint_block")


def test_reference_init_semantics(tiny_model):
    cn = tiny_model.control_model
    sd = cn.state_dict()
    # LoRA up = 0, zero-convs = 0, proj_out = 0, out_layers[-1] = 0 (SURVEY.md §0.4); LoRA down ~ N(0, 1/r)
    assert all(v.abs().max() == 0 for k, v in sd.items() if k.endswith("lora_layer.up.weight"))
    assert all(v.abs().max() == 0 for k, v in sd.items() if k.startswith(("zero_convs", "middle_block_out")))
    assert all(v.abs().max() == 0 for k, v in sd.items() if ".proj_out." in k or ".out_layers.3." in k)
    down = torch.cat([v.flatten() for k, v in sd.items() if k.endswith("lora_layer.down.weight")])
    assert abs(down.std().item() - 1 / 8) < 0.01
    n_lora = sum(1 for k in sd if k.endswith("lora_layer.down.weight"))
    assert n_lora == 82


def test_trainable_filter_matches_reference(g, tiny_model):
    from cldm.cldm_ctrlora_finetune import trainable_parameters
    names = [n for n, _ in trainable_parameters(tiny_model.control_model)]
    assert names == g["trainable_names"]


def test_schedule_and_sampler_tables_bit_exact(g, tiny_model):
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod"):
        assert torch.equal(getattr(tiny_model, k), g[k]), k
    from cldm.ddim_hacked import DDIMSampler
    from ldm.modules.diffusionmodules.util import make_ddim_timesteps
    for S, ts in g["ddim_timesteps"].items():
        assert np.array_equal(make_ddim_timesteps("uniform", S, 1000, verbose=False), ts)
    sampler = DDIMSampler(tiny_model)
    for eta in (0.0, 0.5):
        sampler.make_schedule(50, ddim_eta=eta, verbose=False)  # runs on CPU: host logic only
        ref = g[f"ddim_tables_eta{eta}"]
        for name, ours in (("sigmas", sampler.ddim_sigmas), ("alphas", sampler.ddim_alphas),
                           ("alphas_prev", sampler.ddim_alphas_prev),
                           ("sqrt_one_minus_alphas", sampler.ddim_sqrt_one_minus_alphas)):
            assert np.array_equal(np.asarray(ours, dtype=np.float64), np.asarray(ref[name], dtype=np.float64)), (eta, name)


def test_q_sample_bit_exact(g, tiny_model):
    from oracle import synth
    x = synth.synth_input("x", (g["B"], 4, g["H"], g["H"]), g["seed"])
    noise = synth.synth_input("noise", (g["B"], 4, g["H"], g["H"]), g["seed"])
    assert torch.equal(tiny_model.q_sample(x, g["t"], noise), g["x_noisy"])


def test_lora_fuse_unfuse_api(g):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.lora import LoRACompatibleLinear, LoRALinearLayer
    from oracle import synth
    L = g["lora"]
    lin = LoRACompatibleLinear(16, 24, lora_layer=LoRALinearLayer(16, 24, rank=4))
    lin.load_state_dict(synth.synth_state_dict(L["shapes"], g["seed"], "loratest."))
    lin._fuse_lora(lora_scale=0.7)
    assert lin.lora_layer is None and torch.allclose(lin.weight, L["w_fused_0.7"], atol=1e-6)
    lin._unfuse_lora()
    assert torch.allclose(lin.weight, L["w_unfused"], atol=1e-6)
    bad = LoRACompatibleLinear(4, 4, lora_layer=LoRALinearLayer(4, 4, rank=2))
    bad.lora_layer.up.weight.data.fill_(float("nan"))
    with pytest.raises(ValueError):
        bad._fuse_lora(safe_fusing=True)


def test_switch_lora_order_pretrain_and_inference():
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.cldm_ctrlora_inference import ControlNetInference
    from cldm.cldm_ctrlora_pretrain import ControlNetPretrain
    from cldm.lora import LoRACompatibleLinear
    kw = dict(image_size=32, in_channels=4, hint_channels=3, model_channels=32, attention_resolutions=[4, 2, 1],
              num_res_blocks=2, channel_mult=[1, 2, 4, 4], num_heads=4, use_spatial_transformer=True,
              transformer_depth=1, context_dim=64, legacy=False)
    cn = ControlNetPretrain(lora_rank=4, tasks=["canny", "depth"], **kw)
    assert len(cn.loras_dict["canny"]) == 82
    cn.switch_lora("depth")
    lins = [m for _, m in cn.named_modules() if isinstance(m, LoRACompatibleLinear)]
    assert all(m.lora_layer is cn.loras_dict["depth"][i] for i, m in enumerate(lins))
    assert any(k.startswith("loras_dict.canny.0.down") for k in cn.state_dict())
    ci = ControlNetInference(lora_rank=4, lora_num=2, **kw)
    ci.switch_lora(1)
    lins = [m for _, m in ci.named_modules() if isinstance(m, LoRACompatibleLinear)]
    assert all(m.lora_layer is ci.loras_list[1][i] for i, m in enumerate(lins))
    assert len(ci.zero_convs_list[0]) == 13 and len(ci.norms_list[0]) == 28  # 7 GroupNorm + 21 LayerNorm
    ci.copy_weights_to_switchable()
    keys = ci.state_dict().keys()
    assert any(k.startswith("loras_list.1.") for k in keys) and any(k.startswith("zero_convs_list.0.") for k in keys)


def test_product_fails_loudly_without_gpu(tiny_model):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    x = torch.zeros(1, 4, 16, 16)
    with pytest.raises(Exception) as e:
        tiny_model.apply_model(x, torch.tensor([1]), {"c_crossattn": [torch.zeros(1, 77, 64)], "c_concat": [x]})
    assert "CUDA" in str(e.value) or "cuda" in str(e.value)


def test_style_variant_state_dict_matches_reference():
    """IP-Adapter / style variant (cldm/cldm_style.py, ldm/modules/attention_ip.py): the UNet's state dict has the
    reference's keys, shapes and ORDER (`ip_scale` buffer before the attention's children, to_k_ip / to_v_ip between to_v
    and to_out), the ControlNet is the plain inference one, and a [text, ip] context fails loudly without a GPU."""
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    g = torch.load(os.path.join(GOLD, "tiny_style_golden.pt"), weights_only=False)
    model = create_model(os.path.join(GOLD, "tiny_style.yaml"), init_weights=False)
    unet_sd = model.model.diffusion_model.state_dict()
    assert list(unet_sd.keys()) == g["unet_key_order"]
    assert {k: tuple(v.shape) for k, v in unet_sd.items()} == g["unet_shapes"]
    assert {k: tuple(v.shape) for k, v in model.control_model.state_dict().items()} == g["control_shapes"]
    ip_keys = [k for k in unet_sd if k.endswith("ip_scale")]
    assert ip_keys == g["ip_scale_keys"] and len(ip_keys) == 16
    assert not any("_ip" in k for k in model.control_model.state_dict())
    from ldm.modules.attention_ip import IPCrossAttention
    n_ip = sum(isinstance(m, IPCrossAttention) for m in model.model.diffusion_model.modules())
    assert n_ip == 16  # every attn2 of the UNet, no attn1
    if not torch.cuda.is_available():
        x = torch.zeros(1, 4, 16, 16)
        with pytest.raises(Exception):
            model.apply_model(x, torch.tensor([1]), {"c_crossattn": [torch.zeros(1, 77, 64)], "c_concat": [x],
                                                    "c_ip": [torch.zeros(1, 4, 64)]})
