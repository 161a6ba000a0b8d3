"""Generate tests/golden/*.pt by running the UNMODIFIED reference (/root/reference) in this container.

    python tools/make_golden.py            # tiny config (committed fixture, ~300 KB)
    python tools/make_golden.py --full     # SD1.5-size eps for one image (committed fixture, ~70 KB; takes minutes)
    python tools/make_golden.py --accum    # gradient accumulation windows, finetune and pretrain (tiny config)
    python tools/make_golden.py --resume   # AdamW state of a checkpoint and the steps after it (tiny config)
    python tools/make_golden.py --dpm      # DPMSolverSampler samples (tiny configs) and host schedule (SD1.5 alphas)
    python tools/make_golden.py --dpm-full # DPMSolverSampler samples at SD1.5 size, batch 1 (about a minute)

The reference cannot travel to the GPU box; these fixtures can.  Weights/inputs are regenerated from names by
oracle/synth.py, so the fixtures hold only key/shape lists and outputs.
"""
import argparse
import copy
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from tools import ref_shims  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests"))
from golden_io import save_golden  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def build_reference(yaml_path, seed):
    ref_shims.install()
    from cldm.model import create_model  # the reference's own factory (cldm/model.py:24-28)
    torch.manual_seed(0)
    model = create_model(yaml_path)
    model.eval()
    for sub, prefix in ((model.control_model, "control_model."), (model.model.diffusion_model, "model.diffusion_model.")):
        shapes = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
        sub.load_state_dict(synth.synth_state_dict(shapes, seed, prefix), strict=True)
    return model


def shapes_of(mod):
    return {k: tuple(v.shape) for k, v in mod.state_dict().items()}


def tiny(seed=0):
    yaml_path = os.path.join(GOLD, "tiny_finetune.yaml")
    model = build_reference(yaml_path, seed)
    cn, unet = model.control_model, model.model.diffusion_model
    B, H = 2, 16
    x = synth.synth_input("x", (B, 4, H, H), seed)
    hint = synth.synth_input("hint", (B, 4, H, H), seed)
    ctx = synth.synth_input("ctx", (B, 77, 64), seed)
    noise = synth.synth_input("noise", (B, 4, H, H), seed)
    t = torch.tensor([981, 21], dtype=torch.long)
    g = {"seed": seed, "B": B, "H": H, "t": t,
         "control_shapes": shapes_of(cn), "unet_shapes": shapes_of(unet),
         "control_key_order": list(cn.state_dict().keys()), "unet_key_order": list(unet.state_dict().keys())}

    with torch.no_grad():
        control = cn(hint=hint, timesteps=t, context=ctx)
        g["control"] = [c.clone() for c in control]
        g["eps"] = unet(x=x, timesteps=t, context=ctx, control=[c.clone() for c in control], only_mid_control=False)
        g["eps_nocontrol"] = unet(x=x, timesteps=t, context=ctx, control=None, only_mid_control=False)
        g["eps_midonly"] = unet(x=x, timesteps=t, context=ctx, control=[c.clone() for c in control], only_mid_control=True)
        scales = [0.5 + 0.1 * i for i in range(13)]
        g["control_scales"] = scales
        g["eps_scaled"] = unet(x=x, timesteps=t, context=ctx, control=[c * s for c, s in zip(control, scales)],
                               only_mid_control=False)
        # apply_model through the reference's own method, VAE stage bypassed (parity boundary = post-VAE)
        model.encode_first_stage = lambda h: h
        model.get_first_stage_encoding = lambda h: h
        g["eps_apply_model"] = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [hint]})

    # training step: q_sample -> apply_model -> loss -> grads of the optimizer's parameter set
    x_noisy = model.q_sample(x_start=x, t=t, noise=noise)
    g["x_noisy"] = x_noisy.clone()
    for p in model.parameters():
        p.grad = None
    eps = model.apply_model(x_noisy, t, {"c_crossattn": [ctx], "c_concat": [hint]})
    loss_simple = model.get_loss(eps, noise, mean=False).mean([1, 2, 3])
    loss = loss_simple.mean()
    loss.backward()
    g["train_eps"] = eps.detach().clone()
    g["loss"] = loss.detach().clone()
    names = []
    for n, p in cn.named_parameters():  # the filter of configure_optimizers (cldm_ctrlora_finetune.py:88-100)
        if "lora_layer" in n or "zero_convs" in n or "middle_block_out" in n or "norm" in n:
            names.append(n)
    g["trainable_names"] = names
    grads = dict(cn.named_parameters())
    g["grad_norms"] = {n: grads[n].grad.norm().item() for n in names}
    keep = [n for n in names if n.startswith(("zero_convs.0.", "middle_block_out", "input_blocks.1.1.norm",
                                               "input_blocks.1.1.transformer_blocks.0.attn1.to_q.lora_layer",
                                               "input_blocks.1.1.transformer_blocks.0.norm1",
                                               "middle_block.1.transformer_blocks.0.ff.net.2.lora_layer",
                                               "time_embed.0.lora_layer", "input_blocks.4.0.emb_layers.1.lora_layer"))]
    g["grads"] = {n: grads[n].grad.clone() for n in keep}

    # schedules / DDIM (bit-exact material)
    from cldm.ddim_hacked import DDIMSampler
    from ldm.modules.diffusionmodules.util import make_ddim_timesteps, timestep_embedding
    g["betas"] = model.betas.clone()
    g["alphas_cumprod"] = model.alphas_cumprod.clone()
    g["alphas_cumprod_prev"] = model.alphas_cumprod_prev.clone()
    g["sqrt_alphas_cumprod"] = model.sqrt_alphas_cumprod.clone()
    g["sqrt_one_minus_alphas_cumprod"] = model.sqrt_one_minus_alphas_cumprod.clone()
    g["ddim_timesteps"] = {S: make_ddim_timesteps("uniform", S, 1000, verbose=False) for S in (50, 20, 10, 2)}
    g["timestep_embedding"] = timestep_embedding(torch.tensor([0, 1, 21, 500, 981, 999]), 32)
    g["timestep_embedding_320"] = timestep_embedding(torch.tensor([981, 21]), 320)
    sampler = DDIMSampler(model)
    sampler.register_buffer = lambda name, attr: setattr(sampler, name, attr)  # reference hard-codes .to('cuda')
    for eta in (0.0, 0.5):
        sampler.make_schedule(50, ddim_eta=eta, verbose=False)
        g[f"ddim_tables_eta{eta}"] = {
            "sigmas": np.asarray(sampler.ddim_sigmas), "alphas": np.asarray(sampler.ddim_alphas),
            "alphas_prev": np.asarray(sampler.ddim_alphas_prev),
            "sqrt_one_minus_alphas": np.asarray(sampler.ddim_sqrt_one_minus_alphas)}
    # one p_sample_ddim with CFG 7.5 through the reference sampler (eta 0), tiny model as the eps predictor
    sampler.make_schedule(50, ddim_eta=0.0, verbose=False)
    uc_ctx = synth.synth_input("uc_ctx", (B, 77, 64), seed)
    cond = {"c_crossattn": [ctx], "c_concat": [hint]}
    ucond = {"c_crossattn": [uc_ctx], "c_concat": [hint]}
    ts = torch.full((B,), 981, dtype=torch.long)
    with torch.no_grad():
        x_prev, pred_x0 = sampler.p_sample_ddim(x, cond, ts, index=49, unconditional_guidance_scale=7.5,
                                                unconditional_conditioning=ucond)
        g["ddim_step"] = {"x_prev": x_prev, "pred_x0": pred_x0, "index": 49, "scale": 7.5}
        # 4-step sampling loop end-to-end (x_T given): exercises the index/timestep bookkeeping
        samples, inter = sampler.sample(4, B, (4, H, H), cond, verbose=False, eta=0.0, x_T=x,
                                        unconditional_guidance_scale=7.5, unconditional_conditioning=ucond,
                                        log_every_t=1)
        g["ddim_sample4"] = {"samples": samples, "pred_x0_last": inter["pred_x0"][-1], "n_inter": len(inter["x_inter"])}

    # LoRA layer semantics (cldm/lora.py)
    from cldm.lora import LoRACompatibleLinear, LoRALinearLayer
    lin = LoRACompatibleLinear(16, 24, lora_layer=LoRALinearLayer(16, 24, rank=4))
    lsd = synth.synth_state_dict({k: tuple(v.shape) for k, v in lin.state_dict().items()}, seed, "loratest.")
    lin.load_state_dict(lsd)
    xin = synth.synth_input("loratest", (3, 16), seed)
    with torch.no_grad():
        y_unfused = lin(xin)
        lin._fuse_lora(lora_scale=0.7)
        w_fused = lin.weight.clone()
        y_fused = lin(xin)
        lin._unfuse_lora()
        w_unfused = lin.weight.clone()
    g["lora"] = {"shapes": {k: tuple(v.shape) for k, v in lsd.items()}, "y": y_unfused, "w_fused_0.7": w_fused,
                 "y_fused_0.7": y_fused, "w_unfused": w_unfused}
    out = os.path.join(GOLD, "tiny_finetune_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


def full(seed=0):
    """One SD1.5-size apply_model (post-VAE) on the reference: rank-128 finetune config, B=1."""
    t0 = time.time()
    yaml_path = os.path.join(ref_shims.REFERENCE_ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml")
    ref_shims.install()
    from omegaconf import OmegaConf
    from ldm.util import instantiate_from_config
    cfg = OmegaConf.load(yaml_path).model.params
    with torch.device("meta"):  # skip the 160 s of default init over 1.33 B params
        cn = instantiate_from_config(cfg.control_stage_config)
        unet = instantiate_from_config(cfg.unet_config)
    cn.eval(), unet.eval()
    for sub, prefix in ((cn, "control_model."), (unet, "model.diffusion_model.")):
        shapes = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
        sub.to_empty(device="cpu")
        sub.load_state_dict(synth.synth_state_dict(shapes, seed, prefix), strict=True)
    print("built in", time.time() - t0)
    B = 1
    x = synth.synth_input("x", (B, 4, 64, 64), seed)
    hint = synth.synth_input("hint", (B, 4, 64, 64), seed)
    ctx = synth.synth_input("ctx", (B, 77, 768), seed)
    t = torch.tensor([501], dtype=torch.long)
    g = {"seed": seed, "t": t, "control_shapes": shapes_of(cn), "unet_shapes": shapes_of(unet)}
    with torch.no_grad():
        control = cn(hint=hint, timesteps=t, context=ctx)
        g["control_norms"] = [c.norm().item() for c in control]
        g["control_12"] = control[12].clone()
        g["control_0_slice"] = control[0][:, :8].clone()
        g["eps"] = unet(x=x, timesteps=t, context=ctx, control=[c.clone() for c in control], only_mid_control=False)
    out = os.path.join(GOLD, "sd15_rank128_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB", "in", time.time() - t0, "s")


def _variant_yaml(kind):
    """tiny_finetune.yaml re-targeted at the pretrain / inference classes (same topology and widths)."""
    txt = open(os.path.join(GOLD, "tiny_finetune.yaml")).read()
    if kind == "pretrain":
        txt = txt.replace("cldm.cldm_ctrlora_finetune.ControlFinetuneLDM", "cldm.cldm_ctrlora_pretrain.ControlPretrainLDM")
        txt = txt.replace("cldm.cldm_ctrlora_finetune.ControlNetFinetune", "cldm.cldm_ctrlora_pretrain.ControlNetPretrain")
        txt = txt.replace("        ft_with_lora: True\n        lora_rank: 8\n        norm_trainable: True\n",
                          "        lora_rank: 8\n        tasks: [ canny, depth, seg ]\n")
    else:
        txt = txt.replace("cldm.cldm_ctrlora_finetune.ControlFinetuneLDM", "cldm.cldm_ctrlora_inference.ControlInferenceLDM")
        txt = txt.replace("cldm.cldm_ctrlora_finetune.ControlNetFinetune", "cldm.cldm_ctrlora_inference.ControlNetInference")
        txt = txt.replace("        ft_with_lora: True\n        lora_rank: 8\n        norm_trainable: True\n",
                          "        lora_rank: 8\n        lora_num: 2\n")
    assert "ft_with_lora" not in txt
    out = os.path.join(GOLD, f"tiny_{kind}.yaml")
    with open(out, "w") as f:
        f.write(txt)
    return out


def variants(seed=0):
    """Reference outputs of the pretrain / inference LDMs (tiny config): ControlPretrainLDM.apply_model per task,
    ControlInferenceLDM.apply_model with 2 LoRA sets + weights, the pretrain training step (loss, gradient norms of ALL
    control_model parameters = the pretrain optimizer's set, cldm_ctrlora_pretrain.py:174-182), and the sampler's
    encode / decode / stochastic_encode."""
    B, H = 2, 16
    x = synth.synth_input("x", (B, 4, H, H), seed)
    hint = synth.synth_input("hint", (B, 4, H, H), seed)
    hint2 = synth.synth_input("hint2", (B, 4, H, H), seed)
    ctx = synth.synth_input("ctx", (B, 77, 64), seed)
    uc_ctx = synth.synth_input("uc_ctx", (B, 77, 64), seed)
    noise = synth.synth_input("noise", (B, 4, H, H), seed)
    t = torch.tensor([981, 21], dtype=torch.long)
    g = {"seed": seed, "B": B, "H": H, "t": t}

    # ---------------- pretrain
    model = build_reference(_variant_yaml("pretrain"), seed)
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    cn = model.control_model
    g["pretrain_control_shapes"], g["unet_shapes"] = shapes_of(cn), shapes_of(model.model.diffusion_model)
    g["pretrain_key_order"] = list(cn.state_dict().keys())
    with torch.no_grad():
        for task in ("canny", "depth", "seg"):
            g[f"pretrain_eps_{task}"] = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": [hint], "task": task})
        g["pretrain_eps_nocontrol"] = model.apply_model(x, t, {"c_crossattn": [ctx], "c_concat": None, "task": "canny"})
    # training step on task 'depth' (p_losses arithmetic: ddpm.py:885-920)
    x_noisy = model.q_sample(x_start=x, t=t, noise=noise)
    for p in model.parameters():
        p.grad = None
    eps = model.apply_model(x_noisy, t, {"c_crossattn": [ctx], "c_concat": [hint], "task": "depth"})
    loss = model.get_loss(eps, noise, mean=False).mean([1, 2, 3]).mean()
    loss.backward()
    g["pretrain_loss"] = loss.detach().clone()
    g["pretrain_train_eps"] = eps.detach().clone()
    named = list(cn.named_parameters())
    g["pretrain_param_names"] = [n for n, _ in named]
    g["pretrain_grad_norms"] = {n: (p.grad.norm().item() if p.grad is not None else None) for n, p in named}
    keep = ("input_blocks.0.0.weight", "input_blocks.0.0.bias", "input_blocks.1.0.in_layers.2.weight",
            "input_blocks.1.0.out_layers.3.weight", "input_blocks.4.0.emb_layers.1.weight", "input_blocks.4.0.emb_layers.1.bias",
            "input_blocks.3.0.op.weight",
            "input_blocks.4.0.skip_connection.weight", "input_blocks.4.1.proj_in.weight",
            "input_blocks.4.1.transformer_blocks.0.attn1.to_q.weight", "input_blocks.4.1.transformer_blocks.0.attn2.to_k.weight",
            "input_blocks.4.1.transformer_blocks.0.ff.net.0.proj.weight", "input_blocks.4.1.transformer_blocks.0.ff.net.0.proj.bias",
            "input_blocks.4.1.transformer_blocks.0.ff.net.2.weight", "middle_block.0.in_layers.0.weight",
            "middle_block.1.proj_out.weight", "middle_block.2.out_layers.3.bias", "time_embed.0.weight", "time_embed.2.bias",
            "zero_convs.3.0.weight", "middle_block_out.0.bias",
            # the attached task's LoRA layers are reached (and de-duplicated by named_parameters) under `lora_layer`
            "time_embed.0.lora_layer.down.weight", "time_embed.0.lora_layer.up.weight",
            "input_blocks.4.1.transformer_blocks.0.attn1.to_q.lora_layer.down.weight",
            "input_blocks.4.1.transformer_blocks.0.ff.net.2.lora_layer.up.weight")
    grads = dict(named)
    g["pretrain_grads"] = {n: grads[n].grad.clone() for n in keep}

    # ---------------- inference (2 LoRA sets, weights 0.7 / 0.3, control_scales ramp)
    model = build_reference(_variant_yaml("inference"), seed)
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    cn = model.control_model
    g["inference_control_shapes"] = shapes_of(cn)
    g["inference_key_order"] = list(cn.state_dict().keys())
    conds = [{"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [ctx], "c_concat": [hint2]}]
    with torch.no_grad():
        g["inference_eps_default"] = model.apply_model(x, t, conds)          # lora_weights = [0.5, 0.5]
        model.lora_weights = [0.7, 0.3]
        model.control_scales = [0.5 + 0.1 * i for i in range(13)]
        g["inference_eps_weighted"] = model.apply_model(x, t, conds)
        model.control_scales = [1.0] * 13
        for i in (0, 1):
            cn.switch_lora(i)
            g[f"inference_control_{i}"] = [c.clone() for c in cn(hint=hint, timesteps=t, context=ctx)]

    # ---------------- sampler encode / decode / stochastic_encode on the finetune model
    model = build_reference(os.path.join(GOLD, "tiny_finetune.yaml"), seed)
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    from cldm.ddim_hacked import DDIMSampler
    sampler = DDIMSampler(model)
    sampler.register_buffer = lambda name, attr: setattr(sampler, name, attr)
    sampler.make_schedule(10, ddim_eta=0.0, verbose=False)
    cond = {"c_crossattn": [ctx], "c_concat": [hint]}
    ucond = {"c_crossattn": [uc_ctx], "c_concat": [hint]}
    with torch.no_grad():
        # scale 1: the reference's CFG branch of encode() concatenates the cond dicts (:258-260) and cannot run here
        x_enc, out = sampler.encode(x, cond, 4, return_intermediates=2)
        g["encode"] = {"x_encoded": x_enc, "intermediate_steps": out["intermediate_steps"],
                       "n_intermediates": len(out["intermediates"])}
        g["decode"] = sampler.decode(x, cond, 4, unconditional_guidance_scale=3.0, unconditional_conditioning=ucond)
        tt = torch.tensor([3, 7], dtype=torch.long)
        # use_original_steps: the DDIM-table branch gathers from a numpy array in the reference (:289) and raises
        g["stochastic_encode"] = {"t": tt, "out": sampler.stochastic_encode(x, tt, use_original_steps=True, noise=noise)}
    # finetune training step with only_mid_control=True (cldm/cldm.py:39-42: the 12 skip residuals are unused)
    model.only_mid_control = True
    x_noisy = model.q_sample(x_start=x, t=t, noise=noise)
    for p in model.parameters():
        p.grad = None
    eps = model.apply_model(x_noisy, t, cond)
    loss = model.get_loss(eps, noise, mean=False).mean([1, 2, 3]).mean()
    loss.backward()
    names = [n for n, _ in model.control_model.named_parameters()
             if "lora_layer" in n or "zero_convs" in n or "middle_block_out" in n or "norm" in n]
    gr = dict(model.control_model.named_parameters())
    g["midonly_train"] = {"loss": loss.detach().clone(), "eps": eps.detach().clone(),
                          "grad_norms": {n: (gr[n].grad.norm().item() if gr[n].grad is not None else 0.0) for n in names}}
    out = os.path.join(GOLD, "tiny_variants_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


def full_train(seed=0):
    """SD1.5-size training step on the reference (rank-128 finetune config, B = 2, checkpointed autograd): loss and the
    gradient norms of the optimizer's 246 tensors (cldm_ctrlora_finetune.py:88-100) + a few full tensors."""
    t0 = time.time()
    yaml_path = os.path.join(ref_shims.REFERENCE_ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml")
    ref_shims.install()
    from omegaconf import OmegaConf
    from ldm.util import instantiate_from_config
    from oracle import ctrlora_oracle as O
    cfg = OmegaConf.load(yaml_path).model.params
    with torch.device("meta"):
        cn = instantiate_from_config(cfg.control_stage_config)
        unet = instantiate_from_config(cfg.unet_config)
    for sub, prefix in ((cn, "control_model."), (unet, "model.diffusion_model.")):
        shapes = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
        sub.to_empty(device="cpu")
        sub.load_state_dict(synth.synth_state_dict(shapes, seed, prefix), strict=True)
    cn.train(), unet.train()   # checkpoint() only recomputes when parameters require grad; dropout is 0
    print("built in", time.time() - t0, flush=True)
    B = 2
    x0 = synth.synth_input("x", (B, 4, 64, 64), seed)
    hint = synth.synth_input("hint", (B, 4, 64, 64), seed)
    ctx = synth.synth_input("ctx", (B, 77, 768), seed)
    noise = synth.synth_input("noise", (B, 4, 64, 64), seed)
    t = torch.tensor([801, 131], dtype=torch.long)
    sched = O.register_schedule()
    x_noisy = O.q_sample(sched, x0, t, noise)   # bit-exact restatement of ddpm.py:356-359 (pinned by the tiny golden)
    control = cn(hint=hint, timesteps=t, context=ctx)
    eps = unet(x=x_noisy, timesteps=t, context=ctx, control=[c for c in control], only_mid_control=False)
    loss = ((eps - noise) ** 2).mean([1, 2, 3]).mean()   # get_loss('l2', mean=False).mean([1,2,3]).mean(), ddpm.py:902-918
    print("forward", time.time() - t0, flush=True)
    loss.backward()
    print("backward", time.time() - t0, flush=True)
    names = [n for n, _ in cn.named_parameters()
             if "lora_layer" in n or "zero_convs" in n or "middle_block_out" in n or "norm" in n]
    grads = dict(cn.named_parameters())
    g = {"seed": seed, "B": B, "t": t, "loss": loss.detach().clone(), "eps": eps.detach().clone(),
         "trainable_names": names, "grad_norms": {n: grads[n].grad.norm().item() for n in names}}
    keep = [n for n in names if n.startswith(("zero_convs.0.", "middle_block_out.0.bias", "input_blocks.1.1.norm",
                                               "input_blocks.1.1.transformer_blocks.0.attn1.to_q.lora_layer.down",
                                               "input_blocks.8.1.transformer_blocks.0.norm2",
                                               "middle_block.1.transformer_blocks.0.attn2.to_v.lora_layer.up",
                                               "time_embed.0.lora_layer.up"))]
    g["grads"] = {n: grads[n].grad.clone() for n in keep}
    out = os.path.join(GOLD, "sd15_rank128_train_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB", "in", time.time() - t0, "s")


def _vae_image(name, shape, seed):
    """synthetic image in [-1, 1]: smooth-ish so that 512x512 inputs are not pure white noise"""
    x = synth.synth_input(name, shape, seed)
    x = torch.nn.functional.avg_pool2d(x, 3, stride=1, padding=1) * 2.0
    return torch.tanh(x)


def vae(seed=0, full=False):
    """First-stage VAE (reference ldm/models/autoencoder.py:82-91, ldm/modules/diffusionmodules/model.py:452-654):
    encode moments / mode and decode on the tiny config, and (--vae-full) on the SD VAE at 512x512, B = 1."""
    ref_shims.install()
    from omegaconf import OmegaConf
    from ldm.util import instantiate_from_config
    g = {"seed": seed}
    if not full:
        cfg = OmegaConf.load(os.path.join(GOLD, "tiny_finetune.yaml")).model.params.first_stage_config
        B, R = 2, 32
    else:
        cfg = OmegaConf.load(os.path.join(ref_shims.REFERENCE_ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml")).model.params.first_stage_config
        B, R = 1, 512
    torch.manual_seed(0)
    m = instantiate_from_config(cfg).eval()
    shapes = shapes_of(m)
    m.load_state_dict(synth.synth_state_dict(shapes, seed, "first_stage_model."), strict=True)
    g["shapes"], g["key_order"] = shapes, list(m.state_dict().keys())
    img = _vae_image("vae_img", (B, 3, R, R), seed)
    z = synth.synth_input("vae_z", (B, 4, R // 8 if full else R // 2, R // 8 if full else R // 2), seed)
    t0 = time.time()
    with torch.no_grad():
        post = m.encode(img)
        g["moments"] = post.parameters.clone()
        g["mode"] = post.mode().clone()
        torch.manual_seed(123)
        g["sample_seed123"] = post.sample().clone()
        print("encode", time.time() - t0, flush=True)
        dec = m.decode(z)
        print("decode", time.time() - t0, flush=True)
    if full:  # keep the fixture small: a crop, a strided subsample and the norm of the 3 MB image
        g["decode_crop"] = dec[:, :, 192:320, 192:320].clone()
        g["decode_strided"] = dec[:, :, ::8, ::8].clone()
        g["decode_norm"] = dec.norm().item()
    else:
        g["decode"] = dec.clone()
        with torch.no_grad():
            g["roundtrip"] = m.decode(post.mode()).clone()
    out = os.path.join(GOLD, "sd_vae_golden.pt" if full else "tiny_vae_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


def ranks(seed=0):
    """BASELINE.json configs[4] (LoRA rank sweep) at the tiny config: the finetune training step of the reference for LoRA
    ranks 4 (not a multiple of 8: exercises the rank padding of the fold / gradient GEMMs), 16 and 32 -- eps, loss, all 246
    gradient norms."""
    base = open(os.path.join(GOLD, "tiny_finetune.yaml")).read()
    B, H = 2, 16
    x = synth.synth_input("x", (B, 4, H, H), seed)
    hint = synth.synth_input("hint", (B, 4, H, H), seed)
    ctx = synth.synth_input("ctx", (B, 77, 64), seed)
    noise = synth.synth_input("noise", (B, 4, H, H), seed)
    t = torch.tensor([981, 21], dtype=torch.long)
    g = {"seed": seed, "B": B, "H": H, "t": t, "ranks": {}}
    for r in (4, 16, 32):
        path = os.path.join("/tmp", f"tiny_rank{r}.yaml")
        with open(path, "w") as f:
            f.write(base.replace("lora_rank: 8", f"lora_rank: {r}"))
        model = build_reference(path, seed)
        model.encode_first_stage = lambda h: h
        model.get_first_stage_encoding = lambda h: h
        x_noisy = model.q_sample(x_start=x, t=t, noise=noise)
        eps = model.apply_model(x_noisy, t, {"c_crossattn": [ctx], "c_concat": [hint]})
        loss = model.get_loss(eps, noise, mean=False).mean([1, 2, 3]).mean()
        loss.backward()
        names = [n for n, _ in model.control_model.named_parameters()
                 if "lora_layer" in n or "zero_convs" in n or "middle_block_out" in n or "norm" in n]
        gr = dict(model.control_model.named_parameters())
        g["ranks"][r] = {"control_shapes": shapes_of(model.control_model), "eps": eps.detach().clone(), "loss": loss.detach().clone(),
                         "grad_norms": {n: gr[n].grad.norm().item() for n in names}}
        g["unet_shapes"] = shapes_of(model.model.diffusion_model)
    out = os.path.join(GOLD, "tiny_ranks_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


def schedule():
    """Task order produced by the reference's BatchSchedulerSampler for seeded np.random (tests/test_scheduler_cpu.py)."""
    import json
    sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from datasets.multi_task_scheduler import BatchSchedulerSampler
    from torch.utils.data import ConcatDataset, Dataset

    class Fake(Dataset):
        def __init__(self, n):
            self.n = n

        def __len__(self):
            return self.n

        def __getitem__(self, i):
            return i

    cases = []
    for seed, sizes, bs, shuffle in ((0, [40, 40, 40], 8, True), (1, [17, 64, 33, 50], 16, True), (2, [10] * 9, 4, True),
                                     (3, [12, 30], 5, False)):
        tasks = [f"task{i}" for i in range(len(sizes))]
        ds = ConcatDataset([Fake(n) for n in sizes])
        np.random.seed(seed)
        torch.manual_seed(seed)
        idx = list(BatchSchedulerSampler(ds, bs, distributed=False, shuffle=shuffle))
        bounds = np.asarray(ds.cumulative_sizes)
        per_batch = []
        for b0 in range(0, len(idx), bs):
            owners = {int(np.searchsorted(bounds, i, side="right")) for i in idx[b0:b0 + bs]}
            assert len(owners) == 1  # one task per mini-batch
            per_batch.append(tasks[owners.pop()])
        cases.append({"seed": seed, "tasks": tasks, "largest": max(sizes), "batch_size": bs, "shuffle": shuffle,
                      "task_per_batch": per_batch})
    out = os.path.join(GOLD, "task_schedule_golden.json")
    json.dump({"cases": cases}, open(out, "w"), indent=1)
    print("wrote", out)


def style(seed=0):
    """IP-Adapter / style variant (tiny config): cldm.cldm_ctrlora_style_inference.ControlInferenceLDM with the UNet of
    cldm.cldm_style (IPCrossAttention in every attn2, ldm/modules/attention_ip.py:196-289).  apply_model with image-prompt
    tokens at two ip_scale settings (all layers / only some layers, as app/gradio_ctrlora_style_transfer.py:131-171 sets
    them), without image prompt, and without hint (guess mode: control None)."""
    txt = open(os.path.join(GOLD, "tiny_finetune.yaml")).read()
    txt = txt.replace("cldm.cldm_ctrlora_finetune.ControlFinetuneLDM", "cldm.cldm_ctrlora_style_inference.ControlInferenceLDM")
    txt = txt.replace("cldm.cldm_ctrlora_finetune.ControlNetFinetune", "cldm.cldm_ctrlora_style_inference.ControlNetInference")
    txt = txt.replace("cldm.cldm.ControlledUnetModel", "cldm.cldm_style.ControlledUnetModel")
    txt = txt.replace("        ft_with_lora: True\n        lora_rank: 8\n        norm_trainable: True\n",
                      "        lora_rank: 8\n        lora_num: 1\n")
    assert "ft_with_lora" not in txt and "cldm_style" in txt
    yaml_path = os.path.join(GOLD, "tiny_style.yaml")
    with open(yaml_path, "w") as f:
        f.write(txt)
    B, H = 2, 16
    x = synth.synth_input("x", (B, 4, H, H), seed)
    hint = synth.synth_input("hint", (B, 4, H, H), seed)
    ctx = synth.synth_input("ctx", (B, 77, 64), seed)
    ip = synth.synth_input("ip", (B, 4, 64), seed)
    t = torch.tensor([981, 21], dtype=torch.long)
    model = build_reference(yaml_path, seed)
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    unet = model.model.diffusion_model
    g = {"seed": seed, "B": B, "H": H, "t": t, "control_shapes": shapes_of(model.control_model), "unet_shapes": shapes_of(unet),
         "unet_key_order": list(unet.state_dict().keys())}
    scale_keys = [k for k in unet.state_dict() if k.endswith("ip_scale")]
    g["ip_scale_keys"] = scale_keys

    def set_scales(values):
        unet.load_state_dict({k: torch.tensor(v) for k, v in values.items()}, strict=False)

    cond = [{"c_crossattn": [ctx], "c_concat": [hint], "c_ip": [ip]}]
    with torch.no_grad():
        # synth weights give every ip_scale buffer a random value: first the state as loaded
        g["ip_scales_loaded"] = {k: float(unet.state_dict()[k]) for k in scale_keys}
        g["eps_loaded"] = model.apply_model(x, t, cond)
        set_scales({k: 0.8 for k in scale_keys})
        g["eps_all_0.8"] = model.apply_model(x, t, cond)
        some = {k: (1.0 if "output_blocks" in k else 0.0) for k in scale_keys}
        set_scales(some)
        g["ip_scales_some"] = some
        g["eps_some"] = model.apply_model(x, t, cond)
        g["eps_no_ip"] = model.apply_model(x, t, [{"c_crossattn": [ctx], "c_concat": [hint]}])
        g["eps_no_hint"] = model.apply_model(x, t, [{"c_crossattn": [ctx], "c_concat": [None], "c_ip": [ip]}])
    out = os.path.join(GOLD, "tiny_style_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


ACCUM_FT_KEEP = ("zero_convs.0.", "middle_block_out", "input_blocks.1.1.norm",
                 "input_blocks.1.1.transformer_blocks.0.attn1.to_q.lora_layer", "time_embed.0.lora_layer",
                 "middle_block.1.transformer_blocks.0.ff.net.2.lora_layer", "input_blocks.4.0.emb_layers.1.lora_layer")
ACCUM_PT_KEEP = ("input_blocks.0.0.weight", "input_blocks.1.0.in_layers.2.weight", "input_blocks.4.1.proj_in.weight",
                 "input_blocks.4.1.transformer_blocks.0.attn1.to_q.weight", "middle_block.1.proj_out.weight",
                 "time_embed.0.weight", "zero_convs.3.0.weight", "middle_block_out.0.bias",
                 "loras_dict.canny.0.down.weight", "loras_dict.canny.5.up.weight",
                 "loras_dict.depth.0.down.weight", "loras_dict.depth.5.up.weight")


def accum(seed=0, lr=1e-3):
    """Gradient accumulation as Lightning 1.5 runs it (accumulate_grad_batches = k), emulated explicitly with the
    reference's modules: per micro-batch the p_losses arithmetic (ddpm.py:885-920), loss / k, .backward() (gradients add
    into .grad), then ONE torch.optim.AdamW step, which skips parameters whose .grad is None.
      finetune (tiny_finetune.yaml): 3 micro-batches of batch 2, the optimizer set of cldm_ctrlora_finetune.py:88-100;
      pretrain (tiny_pretrain.yaml): a window with tasks [canny, depth, canny], switch_lora per micro-batch inside
      apply_model (cldm_ctrlora_pretrain.py:104), AdamW over control_model.parameters() (:174-182)."""
    B, H = 2, 16
    ts = [[981, 21], [500, 250], [37, 760]]

    def micro(i):
        mk = lambda n, s: synth.synth_input(f"{n}_acc{i}", s, seed)
        return dict(x=mk("x", (B, 4, H, H)), hint=mk("hint", (B, 4, H, H)), ctx=mk("ctx", (B, 77, 64)),
                    noise=mk("noise", (B, 4, H, H)), t=torch.tensor(ts[i], dtype=torch.long))

    def window(model, params, tasks):
        k = len(tasks)
        model.encode_first_stage = lambda h: h
        model.get_first_stage_encoding = lambda h: h
        for p in model.parameters():
            p.grad = None
        losses = []
        for i, task in enumerate(tasks):
            d = micro(i)
            cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
            if task is not None:
                cond["task"] = task
            x_noisy = model.q_sample(x_start=d["x"], t=d["t"], noise=d["noise"])
            eps = model.apply_model(x_noisy, d["t"], cond)
            loss = model.get_loss(eps, d["noise"], mean=False).mean([1, 2, 3]).mean()
            (loss / k).backward()
            losses.append(loss.detach().clone())
        opt = torch.optim.AdamW(params, lr=lr)
        return torch.stack(losses), opt

    g = {"seed": seed, "B": B, "H": H, "t": torch.tensor(ts), "lr": lr}
    # ---------------- finetune
    model = build_reference(os.path.join(GOLD, "tiny_finetune.yaml"), seed)
    cn = model.control_model
    names = [n for n, _ in cn.named_parameters()
             if "lora_layer" in n or "zero_convs" in n or "middle_block_out" in n or "norm" in n]
    named = dict(cn.named_parameters())
    params = [named[n] for n in names]
    losses, opt = window(model, params, [None, None, None])
    keep = [n for n in names if n.startswith(ACCUM_FT_KEEP)]
    ft = {"control_shapes": shapes_of(cn), "unet_shapes": shapes_of(model.model.diffusion_model), "losses": losses,
          "trainable_names": names, "grad_norms": {n: named[n].grad.norm().item() for n in names},
          "grads": {n: named[n].grad.clone() for n in keep}, "before": {n: named[n].detach().clone() for n in keep}}
    opt.step()
    ft["after"] = {n: named[n].detach().clone() for n in keep}
    g["finetune"] = ft
    # ---------------- pretrain
    model = build_reference(os.path.join(GOLD, "tiny_pretrain.yaml"), seed)
    cn = model.control_model
    named = [(n, p) for n, p in cn.named_parameters(remove_duplicate=False) if ".lora_layer." not in n]
    by_name = dict(named)
    tasks = ["canny", "depth", "canny"]
    shapes = shapes_of(cn)  # before switch_lora attaches a set (its aliases would join the state dict)
    losses, opt = window(model, list(cn.parameters()), tasks)
    pt = {"control_shapes": shapes, "tasks": tasks, "losses": losses, "param_names": [n for n, _ in named],
          "grad_norms": {n: (p.grad.norm().item() if p.grad is not None else None) for n, p in named},
          "grads": {n: by_name[n].grad.clone() for n in ACCUM_PT_KEEP},
          "before": {n: by_name[n].detach().clone() for n in ACCUM_PT_KEEP}}
    opt.step()
    pt["after"] = {n: by_name[n].detach().clone() for n in ACCUM_PT_KEEP}
    g["pretrain"] = pt
    out = os.path.join(GOLD, "tiny_accum_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


RESUME_FT_KEEP = ("zero_convs.2.0.weight", "input_blocks.1.1.transformer_blocks.0.attn1.to_q.lora_layer.up.weight",
                  "input_blocks.1.1.transformer_blocks.0.attn1.to_q.lora_layer.down.weight", "input_blocks.1.1.norm.weight",
                  "input_blocks.1.1.norm.bias", "middle_block_out.0.bias")
RESUME_PT_KEEP = ("input_blocks.0.0.weight", "input_blocks.1.0.in_layers.2.weight", "input_blocks.4.0.in_layers.2.weight",
                  "input_blocks.4.1.transformer_blocks.0.attn1.to_q.weight", "input_blocks.1.0.in_layers.0.weight",
                  "zero_convs.3.0.weight", "middle_block_out.0.bias",
                  "loras_dict.canny.0.down.weight", "loras_dict.depth.5.up.weight",
                  "loras_dict.seg.0.down.weight", "loras_dict.seg.5.up.weight")


def resume(seed=0, lr=1e-3):
    """The AdamW state a Lightning checkpoint holds (`optimizer_states[0]` = torch.optim.AdamW.state_dict() over the
    parameter list configure_optimizers builds), and the steps that continue from it, with the reference's modules:
      finetune (tiny_finetune.yaml): one step on micro-batch 0 (the trainable parameters after it and the whole
        optimizer state dict), then a second step on micro-batch 1 (the update of the sampled tensors);
      pretrain (tiny_pretrain.yaml): steps on [canny] then [depth] (index -> name list, which indices have state and
        their `step`, the moments of the sampled tensors, 3x3 convs included), then a third step on [seg] (the update
        of the sampled tensors: base at step 3, seg at step 1).
    Gradients are cleared to None before every step, so a LoRA set no step used gets no state (AdamW skips it)."""
    B, H = 2, 16
    ts = [[981, 21], [500, 250], [37, 760]]

    def micro(i):
        mk = lambda n, s: synth.synth_input(f"{n}_acc{i}", s, seed)
        return dict(x=mk("x", (B, 4, H, H)), hint=mk("hint", (B, 4, H, H)), ctx=mk("ctx", (B, 77, 64)),
                    noise=mk("noise", (B, 4, H, H)), t=torch.tensor(ts[i], dtype=torch.long))

    def step(model, opt, i, task=None):
        model.encode_first_stage = lambda h: h
        model.get_first_stage_encoding = lambda h: h
        opt.zero_grad(set_to_none=True)
        d = micro(i)
        cond = {"c_crossattn": [d["ctx"]], "c_concat": [d["hint"]]}
        if task is not None:
            cond["task"] = task
        x_noisy = model.q_sample(x_start=d["x"], t=d["t"], noise=d["noise"])
        eps = model.apply_model(x_noisy, d["t"], cond)
        loss = model.get_loss(eps, d["noise"], mean=False).mean([1, 2, 3]).mean()
        loss.backward()
        opt.step()
        return loss.detach().clone()

    g = {"seed": seed, "B": B, "H": H, "t": torch.tensor(ts), "lr": lr}
    # ---------------- finetune
    model = build_reference(os.path.join(GOLD, "tiny_finetune.yaml"), seed)
    cn = model.control_model
    names = [n for n, _ in cn.named_parameters()
             if "lora_layer" in n or "zero_convs" in n or "middle_block_out" in n or "norm" in n]
    named = dict(cn.named_parameters())
    opt = torch.optim.AdamW([named[n] for n in names], lr=lr)
    ft = {"control_shapes": shapes_of(cn), "unet_shapes": shapes_of(model.model.diffusion_model),
          "trainable_names": names}
    ft["loss1"] = step(model, opt, 0)
    sd = copy.deepcopy(opt.state_dict())  # state_dict() holds the live tensors: the next step would update them
    ft["param_groups1"] = sd["param_groups"]
    # whole-set entries live at the top level, where save_golden splits a dict entry by entry into part files
    g["ft_params1"] = {n: named[n].detach().clone() for n in names}
    g["ft_state1"] = sd["state"]  # optimizer_states[0]["state"] of a checkpoint taken after step 1
    ft["loss2"] = step(model, opt, 1)
    ft["after2"] = {n: named[n].detach().clone() for n in RESUME_FT_KEEP}
    g["finetune"] = ft
    # ---------------- pretrain
    model = build_reference(os.path.join(GOLD, "tiny_pretrain.yaml"), seed)
    cn = model.control_model
    shapes = shapes_of(cn)  # before switch_lora attaches a set
    params = list(cn.parameters())  # configure_optimizers (cldm_ctrlora_pretrain.py:174-182), before any switch_lora
    name_of = {id(p): n for n, p in cn.named_parameters()}
    index_names = [name_of[id(p)] for p in params]
    opt = torch.optim.AdamW(params, lr=lr)
    by_name = dict(zip(index_names, params))
    pt = {"control_shapes": shapes, "index_names": index_names}
    pt["losses"] = torch.stack([step(model, opt, 0, "canny"), step(model, opt, 1, "depth")])
    sd = copy.deepcopy(opt.state_dict())
    pt["steps"] = {i: int(s["step"]) for i, s in sd["state"].items()}
    pt["param_group"] = {k: v for k, v in sd["param_groups"][0].items() if k != "params"}
    pt["moments"] = {n: {k: sd["state"][index_names.index(n)][k].clone() for k in ("exp_avg", "exp_avg_sq")}
                     for n in RESUME_PT_KEEP if index_names.index(n) in sd["state"]}
    pt["before3"] = {n: by_name[n].detach().clone() for n in RESUME_PT_KEEP}
    pt["loss3"] = step(model, opt, 2, "seg")
    pt["after3"] = {n: by_name[n].detach().clone() for n in RESUME_PT_KEEP}
    pt["steps3"] = {i: int(s["step"]) for i, s in opt.state_dict()["state"].items()}
    g["pretrain"] = pt
    out = os.path.join(GOLD, "tiny_resume_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


DPM_TINY_STEPS = (4, 5, 16)            # both sides of lower_order_final's `steps < 15` switch
DPM_SCHEDULE_STEPS = (4, 5, 10, 16, 20, 25)


def _sd15_reference_ldm(seed):
    """The reference's ControlFinetuneLDM at SD1.5 size (rank-128 finetune config) with synthetic weights.  torch.nn.init
    is stubbed while it is built: the default init of 1.33 B parameters takes minutes and is overwritten anyway."""
    from unittest import mock
    ref_shims.install()
    from cldm.model import create_model
    yaml_path = os.path.join(ref_shims.REFERENCE_ROOT, "configs", "ctrlora_finetune_sd15_rank128.yaml")
    keep = lambda t, *a, **k: t
    with mock.patch.multiple(torch.nn.init, kaiming_uniform_=keep, uniform_=keep, normal_=keep, xavier_uniform_=keep):
        model = create_model(yaml_path)
    model.eval()
    for sub, prefix in ((model.control_model, "control_model."), (model.model.diffusion_model, "model.diffusion_model.")):
        shapes = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
        sub.load_state_dict(synth.synth_state_dict(shapes, seed, prefix), strict=True)
    return model


def _dpm_reference_sample(model, x_T, steps, cond, ucond, scale):
    """DPMSolverSampler.sample (ldm/models/diffusion/dpm_solver/sampler.py:60-87) with the reference's own
    NoiseScheduleVP, model_wrapper and DPM_Solver and the arguments of :72-85, on the reference model's apply_model.
    Two substitutions where the reference cannot run on ControlLDM conditioning (DESIGN.md §7):
      * the `.shape` check of the conditioning (:51-58) is skipped (c_concat is a list; the inference model's
        conditioning is a list of dicts);
      * with guidance, model_wrapper's classifier-free branch `torch.cat`s the cond dicts (dpm_solver.py:308-310), so
        model_wrapper(guidance_type="uncond") gets a model that evaluates apply_model on cond and on uncond and combines
        them with :312's formula, e_u + scale * (e_c - e_u).  Without guidance the classifier-free branch runs as is."""
    from ldm.models.diffusion.dpm_solver.dpm_solver import DPM_Solver, NoiseScheduleVP, model_wrapper
    ns = NoiseScheduleVP('discrete', alphas_cumprod=model.alphas_cumprod.clone().detach().to(torch.float32))
    if ucond is None or scale == 1.:
        model_fn = model_wrapper(lambda x, t, c: model.apply_model(x, t, c), ns, model_type="noise",
                                 guidance_type="classifier-free", condition=cond, unconditional_condition=ucond,
                                 guidance_scale=scale)
    else:
        def guided(x, t):
            e_c, e_u = model.apply_model(x, t, cond), model.apply_model(x, t, ucond)
            return e_u + scale * (e_c - e_u)
        model_fn = model_wrapper(guided, ns, model_type="noise", guidance_type="uncond")
    dpm_solver = DPM_Solver(model_fn, ns, predict_x0=True, thresholding=False)
    with torch.no_grad():
        return dpm_solver.sample(x_T.clone(), steps=steps, skip_type="time_uniform", method="multistep", order=2,
                                 lower_order_final=True)


def _dpm_schedule_record(alphas_cumprod, steps):
    """Per step of the reference's multistep loop (dpm_solver.py:1044-1074), from its own objects at batch 1: the step
    time, the model input time the wrapper hands apply_model, alpha / sigma / lambda there, and the update coefficients
    read back from multistep_dpm_solver_update through probe inputs: x = 1 -> c_x; m = m_prev = 1 -> -c_m;
    m = 0, m_prev = -1 -> -(c_d * inv_r0)."""
    from ldm.models.diffusion.dpm_solver.dpm_solver import DPM_Solver, NoiseScheduleVP, model_wrapper
    ns = NoiseScheduleVP('discrete', alphas_cumprod=alphas_cumprod)
    seen = []

    def record(x, t_input):
        seen.append(t_input.clone())
        return torch.zeros_like(x)
    dpm = DPM_Solver(model_wrapper(record, ns, model_type="noise", guidance_type="uncond"), ns, predict_x0=True)
    dpm.sample(torch.zeros(1, 1), steps=steps, skip_type="time_uniform", method="multistep", order=2, lower_order_final=True)
    ts = dpm.get_time_steps(skip_type="time_uniform", t_T=ns.T, t_0=1. / ns.total_N, N=steps, device="cpu")
    one, zero = torch.ones(1, 1), torch.zeros(1, 1)
    rec = {"t": [], "model_time": [float(v[0]) for v in seen], "alpha": [], "sigma": [], "lambda": [], "order": [],
           "c_x": [], "neg_c_m": [], "neg_c_d_inv_r0": []}
    for i in range(steps):
        s = ts[i].expand(1)
        order = 1 if i == 0 else (min(2, steps - i) if steps < 15 else 2)
        rec["t"].append(float(s[0]))
        rec["alpha"].append(float(ns.marginal_alpha(s)[0]))
        rec["sigma"].append(float(ns.marginal_std(s)[0]))
        rec["lambda"].append(float(ns.marginal_lambda(s)[0]))
        rec["order"].append(order)
        t_prev = [ts[max(i - 1, 0)].expand(1), s]
        upd = lambda x, m1, m0: float(dpm.multistep_dpm_solver_update(x, [m1, m0], t_prev, ts[i + 1].expand(1), order)[0, 0])
        rec["c_x"].append(upd(one, zero, zero))
        rec["neg_c_m"].append(upd(zero, one, one))
        rec["neg_c_d_inv_r0"].append(upd(zero, -one, zero) if order == 2 else 0.0)
    return rec


def dpm(seed=0, full=False):
    """The reference's DPMSolverSampler (see _dpm_reference_sample): final samples from a seeded x_T.
      default: tiny finetune config, steps 4 / 5 / 16, with and without CFG 7.5; tiny 2-LoRA inference config, steps 5
        with CFG 7.5 and lora_weights [0.7, 0.3]; and the host schedule for the SD1.5 alphas_cumprod
        (_dpm_schedule_record, steps 4 / 5 / 10 / 16 / 20 / 25);
      --dpm-full: SD1.5 rank 128, batch 1, 64x64 latent, steps 3 with CFG 7.5 (order-1 start, order 2, order-1 end)."""
    if full:
        model = _sd15_reference_ldm(seed)
        model.encode_first_stage = lambda h: h
        model.get_first_stage_encoding = lambda h: h
        B, R = 1, 64
        x_T = synth.synth_input("dpm_xT", (B, 4, R, R), seed)
        hint = synth.synth_input("hint", (B, 4, R, R), seed)
        ctx, uc = synth.synth_input("ctx", (B, 77, 768), seed), synth.synth_input("uc_ctx", (B, 77, 768), seed)
        cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
        t0 = time.time()
        g = {"seed": seed, "B": B, "R": R, "steps": 3, "scale": 7.5,
             "samples": _dpm_reference_sample(model, x_T, 3, cond, ucond, 7.5)}
        print("sampled in", time.time() - t0, "s")
        out = os.path.join(GOLD, "sd15_dpm_golden.pt")
        save_golden(g, out)
        print("wrote", out, os.path.getsize(out) // 1024, "KiB")
        return
    B, H = 2, 16
    x_T = synth.synth_input("dpm_xT", (B, 4, H, H), seed)
    hint, hint2 = synth.synth_input("hint", (B, 4, H, H), seed), synth.synth_input("hint2", (B, 4, H, H), seed)
    ctx, uc = synth.synth_input("ctx", (B, 77, 64), seed), synth.synth_input("uc_ctx", (B, 77, 64), seed)
    g = {"seed": seed, "B": B, "H": H, "scale": 7.5, "finetune": {}, "inference": {}}
    model = build_reference(os.path.join(GOLD, "tiny_finetune.yaml"), seed)
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    cond, ucond = {"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint]}
    for S in DPM_TINY_STEPS:
        g["finetune"][(S, 1.0)] = _dpm_reference_sample(model, x_T, S, cond, None, 1.0)
        g["finetune"][(S, 7.5)] = _dpm_reference_sample(model, x_T, S, cond, ucond, 7.5)
    model = build_reference(_variant_yaml("inference"), seed)
    model.encode_first_stage = lambda h: h
    model.get_first_stage_encoding = lambda h: h
    model.lora_weights = [0.7, 0.3]
    g["inference_lora_weights"] = [0.7, 0.3]
    conds = [{"c_crossattn": [ctx], "c_concat": [hint]}, {"c_crossattn": [ctx], "c_concat": [hint2]}]
    uconds = [{"c_crossattn": [uc], "c_concat": [hint]}, {"c_crossattn": [uc], "c_concat": [hint2]}]
    g["inference"][(5, 7.5)] = _dpm_reference_sample(model, x_T, 5, conds, uconds, 7.5)
    # host schedule for the SD1.5 alphas_cumprod (the configs' linear schedule, 0.00085 .. 0.012)
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    betas = make_beta_schedule("linear", 1000, linear_start=0.00085, linear_end=0.012)
    ac = torch.tensor(np.cumprod(1. - betas, axis=0), dtype=torch.float32)
    g["sd15_alphas_cumprod"] = ac
    g["schedule"] = {S: _dpm_schedule_record(ac, S) for S in DPM_SCHEDULE_STEPS}
    out = os.path.join(GOLD, "tiny_dpm_golden.pt")
    save_golden(g, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--dpm", action="store_true")
    ap.add_argument("--dpm-full", action="store_true")
    ap.add_argument("--accum", action="store_true")
    ap.add_argument("--full", action="store_true")
    ap.add_argument("--variants", action="store_true")
    ap.add_argument("--full-train", action="store_true")
    ap.add_argument("--schedule", action="store_true")
    ap.add_argument("--ranks", action="store_true")
    ap.add_argument("--vae", action="store_true")
    ap.add_argument("--vae-full", action="store_true")
    ap.add_argument("--style", action="store_true")
    ap.add_argument("--resume", action="store_true")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    if a.full:
        full()
    elif a.variants:
        variants()
    elif a.full_train:
        full_train()
    elif a.schedule:
        schedule()
    elif a.ranks:
        ranks()
    elif a.vae:
        vae()
    elif a.vae_full:
        vae(full=True)
    elif a.style:
        style()
    elif a.accum:
        accum()
    elif a.resume:
        resume()
    elif a.dpm:
        dpm()
    elif a.dpm_full:
        dpm(full=True)
    else:
        tiny()
