"""The IP-Adapter image encoder on the sm_90a kernels: the new kernels (patch gather, embedding assembly, exact GELU)
against fp32 torch, the attention kernel at the encoder's 257 x 257 d_head-80 shape, the tiny and ViT-H image encoders,
the image-prompt projection and the text towers against the fixture (tests/golden/clip_vision_golden.pt,
`tools/make_clip_vision_golden.py`: transformers and the reference app's ImageProjModel in fp32) and against transformers
on the GPU at another batch size, the fp16 module as the style app builds it, weight reloads, and DDIM sampling of the
tiny style model with our image-prompt tokens.  Errors are printed under `pytest -s`, with transformers' own fp16 error
(what the reference app runs) beside ours."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import clip_vision_golden as cvg

pytestmark = pytest.mark.gpu
ROOT = cvg.ROOT

# Norm-relative error bounds (||got - ref|| / ||ref||) against the fp32 fixture, about 20 % above what an H100 measured
# (NVIDIA H100 80GB HBM3, 700 W; the measured value in the comment).  GEMM operands and attention are fp16 with fp32
# accumulation, the residual stream and LayerNorm statistics fp32.
# transformers' own eager fp16 run (the reference app's setting) measured 8.0e-4 (tiny) and 1.59e-3 (ViT-H) on
# image_embeds, 8.7e-4 and 1.73e-3 on text_embeds, against the same fixture.
TOL = {
    # measured against the fixture / against transformers fp32 on the GPU at batch 3 (text: batch 4)
    "vision_tiny": 4.9e-4,          # image_embeds: 3.86e-4 / 4.10e-4
    "vision_tiny_hidden": 5.6e-4,   # last_hidden_state: 4.69e-4 / 4.67e-4
    "vision_sd15": 8.7e-4,          # image_embeds, 32 layers: 7.05e-4 / 7.22e-4
    "vision_sd15_hidden": 8.5e-4,   # last_hidden_state: - / 7.09e-4
    "tokens_tiny": 5.2e-4,          # ImageProjModel cond tokens: 4.32e-4 (uncond, the bias through LayerNorm: 8e-8)
    "tokens_sd15": 8.9e-4,          # 7.44e-4
    "text_tiny": 8.3e-4,            # text_embeds: 6.62e-4 / 6.95e-4, rows of real tokens 6.66e-4
    "text_sd15": 1.19e-3,           # 9.24e-4 / 9.90e-4, rows of real tokens 8.63e-4
}
# fp16 parameters and outputs, as the style app runs the modules (ViT-H, against the fp32 fixture)
TOL16 = {"image_embeds": 1.03e-3,   # 8.59e-4
         "text_embeds": 1.28e-3,    # 1.06e-3
         "tokens": 1.13e-3,         # 9.41e-4
         "uncond": 4.5e-4}          # 3.76e-4: fp16 bias and LayerNorm parameters
ATTN_TOL = 3.2e-4     # ctrlora_attention_f16 at 257 x 257, d 80, 16 heads: 2.69e-4 at batch 1 and 4
LAST_KEY_TOL = 5e-3   # its key 256 (alone in the last key tile) on its own: 4.18e-3
SAMPLE_TOL = 4.3e-3   # DDIM sample with our c_ip against the sample with the fixture's c_ip: 3.61e-3


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(scope="module")
def g():
    return cvg.load()


def vision(which, seed=cvg.SEED):
    from ctrlora_b200.image_encoder import CLIPVisionModelWithProjection
    m = CLIPVisionModelWithProjection(cvg.VISION[which])
    m.load_state_dict(cvg.weights(m, "vision", seed), strict=True)
    return m.cuda()


def image_proj(which):
    from ctrlora_b200.image_encoder import ImageProjModel
    p = ImageProjModel(**cvg.PROJ[which])
    p.load_state_dict(cvg.weights(p, "proj"), strict=True)
    return p.cuda()


def text(which, g):
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection
    cfg = g["text_" + which]["config"]
    m = CLIPTextModelWithProjection(cfg)
    m.load_state_dict(cvg.weights(m, "text"), strict=True)
    return m.cuda()


def hf_vision(which, dtype=torch.float32):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    m = CLIPVisionModelWithProjection(CLIPVisionConfig(**cvg.VISION[which])).eval()
    m.load_state_dict(cvg.weights(m, "vision"), strict=True)
    return m.to("cuda", dtype=dtype)


def hf_text(cfg, dtype=torch.float32):
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    m = CLIPTextModelWithProjection(CLIPTextConfig(**cfg)).eval()
    m.load_state_dict(cvg.weights(m, "text"), strict=True)
    return m.to("cuda", dtype=dtype)


# ------------------------------------------------------------------------------------------------ the new kernels
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_patch_gather_is_the_conv(dtype):
    from ctrlora_b200 import ops, prepare
    gen = torch.Generator(device="cuda").manual_seed(3)
    px = torch.randn((3, 3, 224, 224), device="cuda", generator=gen).to(dtype)
    w = torch.randn((160, 3, 14, 14), device="cuda", generator=gen) / 588 ** 0.5
    rows = ops.clip_patch_gather(px, 14, 592)
    assert rows.shape == (3 * 256, 592) and (rows[:, 588:] == 0).all()
    assert torch.equal(rows, ops.clip_patch_gather(px, 14, 592))
    # the gather itself is exact: the (c, kh, kw) unfold of the patches
    unfold = px.float().view(3, 3, 16, 14, 16, 14).permute(0, 2, 4, 1, 3, 5).reshape(3 * 256, 588)
    assert torch.equal(rows[:, :588], unfold.half())
    w16 = torch.zeros((160, 1, 592), device="cuda", dtype=torch.float16)
    w16[:, :, :588] = prepare.linear_weight(w.reshape(160, 588))
    got = ops.gemm(rows, w16, out_f32=True)
    ref = F.conv2d(px.float().half().float(), w.half().float(), stride=14).flatten(2).transpose(1, 2).reshape(-1, 160)
    err = rel(got, ref)
    print(f"patch embedding ({dtype}) vs F.conv2d: rel err {err:.2e}")
    assert err < 6e-7  # same fp16 operands, fp32 accumulation in another order: 4.99e-7 measured


def test_embedding_assembly_and_pre_layernorm():
    from ctrlora_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(4)
    b, p, c = 3, 256, 1280
    patch = torch.randn((b * p, c), device="cuda", generator=gen)
    cls = torch.randn(c, device="cuda", generator=gen)
    pos = torch.randn((p + 1, c), device="cuda", generator=gen)
    gamma, beta = 1 + 0.1 * torch.randn(c, device="cuda", generator=gen), 0.1 * torch.randn(c, device="cuda", generator=gen)
    h = ops.clip_vision_embed(patch, cls, pos, b)
    ref = torch.cat([cls.expand(b, 1, c), patch.view(b, p, c)], dim=1) + pos
    assert torch.equal(h.view(b, p + 1, c), ref)  # one fp32 add, as transformers
    y = ops.layernorm_rows(h, gamma, beta, 1e-5, out_f32=True)
    err = rel(y, F.layer_norm(ref, (c,), gamma, beta, 1e-5).view(-1, c))
    print(f"pre_layrnorm vs F.layer_norm: rel err {err:.2e}")
    assert err < 7e-8  # 5.82e-8 measured
    assert torch.equal(ops.clip_vision_embed(patch, cls, pos, b), h)


def test_exact_gelu():
    from ctrlora_b200 import ops
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    x = torch.cat([torch.tensor([10.0, -10.0, 6e-8, -6e-8, 3e-5, -3e-5]).half(), bits[torch.isfinite(bits)]])
    x = x[: x.numel() // 8 * 8].cuda().contiguous()
    got = ops.gelu_(x.clone())
    assert torch.equal(got, ops.gelu_(x.clone()))
    ref = F.gelu(x.float())
    err = (got.float() - ref).abs()
    # one fp16 rounding of the result plus the erf approximation's 1.5e-7 (|x| / 2 times it)
    bound = ref.abs() * 2.0 ** -10 + 6e-8 + 1e-7 * x.float().abs()
    print(f"gelu over {x.numel()} fp16 values: max abs err {err.max():.2e}, worst err / bound {(err / bound).max():.3f}")
    assert (err <= bound).all()
    sub = x.float().abs() < 6.1e-5  # fp16 subnormals: gelu(x) = x / 2 to fp16 rounding
    assert (err[sub] <= 6e-8).all()


# ------------------------------------------------------------------------------------------------ attention at 257 tokens
@pytest.mark.parametrize("batch", [1, 4])
def test_attention_257_tokens_d80(batch):
    from ctrlora_b200 import ops
    heads, d, n = 16, 80, 257
    gen = torch.Generator(device="cuda").manual_seed(batch)
    q, k, v = (torch.randn((batch, n, heads * d), device="cuda", generator=gen).half() for _ in range(3))
    vt = torch.full((batch, heads, d, 264), float("nan"), device="cuda", dtype=torch.float16)  # padding is never read
    vt[..., :n] = v.view(batch, n, heads, d).permute(0, 2, 3, 1)
    out = ops.attention(q.view(-1, heads * d), k.view(-1, heads * d), vt, batch, heads, n, n, d)
    again = ops.attention(q.view(-1, heads * d), k.view(-1, heads * d), vt, batch, heads, n, n, d)
    assert torch.equal(out, again)
    qf, kf, vf = (t.float().view(batch, n, heads, d).transpose(1, 2) for t in (q, k, v))
    p = (qf @ kf.transpose(-1, -2) / d ** 0.5).softmax(-1)
    ref = (p @ vf).transpose(1, 2).reshape(batch * n, heads * d)
    err = rel(out, ref)
    # the last key tile holds one valid key: its weight must be there (and nothing of the NaN padding)
    last = (p[..., -1:] @ vf[..., -1:, :]).transpose(1, 2).reshape(batch * n, heads * d)
    err_last = rel(out.float() - (ref - last), last)
    print(f"attention 257x257 d80 batch {batch}: rel err {err:.2e}; key 256 alone {err_last:.2e}")
    assert torch.isfinite(out).all() and err < ATTN_TOL and err_last < LAST_KEY_TOL


# ------------------------------------------------------------------------------------------------ the models
@pytest.mark.parametrize("which", ["tiny", "sd15"])
def test_vision_against_fixture(g, which):
    ref = g["vision_" + which]
    model, proj = vision(which), image_proj(which)
    px = cvg.pixels(cvg.BATCH)
    out = model(px)
    emb = out.image_embeds
    assert emb.dtype == torch.float32 and emb.shape == ref["image_embeds"].shape
    e = {"embeds": rel(emb, ref["image_embeds"])}
    tok, untok = proj(emb), proj(torch.zeros_like(emb))
    e["tokens"] = rel(tok, ref["tokens"])
    e["uncond"] = rel(untok, ref["uncond_tokens"])
    if which == "tiny":
        e["hidden"] = rel(out.last_hidden_state, ref["last_hidden_state"])
    hf16 = hf_vision(which, torch.float16)
    with torch.no_grad():
        e16 = rel(hf16(px.cuda().half()).image_embeds, ref["image_embeds"])
    print(f"vision {which}: " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()) + f" (transformers fp16 embeds {e16:.3e})")
    assert e["embeds"] < TOL["vision_" + which]
    assert e["tokens"] < TOL["tokens_" + which] and e["uncond"] < 1e-7  # 8.4e-8 measured
    if which == "tiny":
        assert e["hidden"] < TOL["vision_tiny_hidden"]
    assert torch.equal(model(px.cuda()).image_embeds, emb)  # host or device pixels, same bits


@pytest.mark.parametrize("which", ["tiny", "sd15"])
def test_vision_against_transformers_batch3(which):
    model, hf = vision(which), hf_vision(which)
    px = cvg.pixels(3, seed=5).cuda()
    with torch.no_grad():
        ref = hf(px)
    out = model(px)
    e, eh = rel(out.image_embeds, ref.image_embeds), rel(out.last_hidden_state, ref.last_hidden_state)
    print(f"vision {which} vs transformers at batch 3: embeds {e:.3e}, last_hidden_state {eh:.3e}")
    assert e < TOL["vision_" + which] and eh < TOL[f"vision_{which}_hidden"]


@pytest.mark.parametrize("which", ["tiny", "sd15"])
def test_text_against_fixture_and_transformers(g, which):
    ref = g["text_" + which]
    model = text(which, g)
    out = model(ref["ids"], attention_mask=ref["attention_mask"])
    err = rel(out.text_embeds, ref["text_embeds"])
    assert torch.equal(model(ref["ids"]).text_embeds, out.text_embeds)  # padded keys never reach the EOS row
    hf16 = hf_text(ref["config"], torch.float16)
    with torch.no_grad():
        e16 = rel(hf16(input_ids=ref["ids"].cuda(), attention_mask=ref["attention_mask"].cuda()).text_embeds, ref["text_embeds"])
    # another batch: the prompts reversed plus one, against transformers on the GPU
    ids = torch.cat([ref["ids"].flip(0), ref["ids"][:1]])
    mask = torch.cat([ref["attention_mask"].flip(0), ref["attention_mask"][:1]])
    hf = hf_text(ref["config"])
    with torch.no_grad():
        r = hf(input_ids=ids.cuda(), attention_mask=mask.cuda())
    o = model(ids, attention_mask=mask)
    e2 = rel(o.text_embeds, r.text_embeds)
    keep = mask.bool().cuda()
    eh = rel(o.last_hidden_state[keep], r.last_hidden_state[keep])
    print(f"text {which}: text_embeds {err:.3e} (transformers fp16 {e16:.3e}); vs transformers at batch 4: {e2:.3e}, "
          f"unpadded rows {eh:.3e}")
    assert max(err, e2, eh) < TOL["text_" + which]


def test_fp16_module_as_the_app_builds_it(g, tmp_path):
    """app/gradio_ctrlora_style_transfer.py:385-409 with the imports swapped"""
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection, CLIPVisionModelWithProjection, ImageProjModel
    d = str(tmp_path)
    src = CLIPVisionModelWithProjection(cvg.VISION["sd15"])
    from safetensors.torch import save_file
    save_file(cvg.weights(src, "vision"), os.path.join(d, "model.safetensors"))
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(cvg.VISION["sd15"], f)
    del src
    image_encoder = CLIPVisionModelWithProjection.from_pretrained(d).to("cuda", dtype=torch.float16)
    clip_image = cvg.pixels(cvg.BATCH)
    clip_image_embeds = image_encoder(clip_image.to("cuda", dtype=torch.float16)).image_embeds
    assert clip_image_embeds.dtype == torch.float16
    ref = g["vision_sd15"]
    e_emb = rel(clip_image_embeds, ref["image_embeds"])
    text_encoder = CLIPTextModelWithProjection(g["text_sd15"]["config"])
    text_encoder.load_state_dict(cvg.weights(text_encoder, "text"))
    text_encoder = text_encoder.to("cuda", dtype=torch.float16)
    tokens = {"input_ids": g["text_sd15"]["ids"][1:2].cuda(), "attention_mask": g["text_sd15"]["attention_mask"][1:2].cuda()}
    neg_content_emb = text_encoder(**tokens).text_embeds
    assert neg_content_emb.dtype == torch.float16
    e_txt = rel(neg_content_emb, g["text_sd15"]["text_embeds"][1:2])
    image_proj = ImageProjModel().to("cuda", dtype=torch.float16)
    image_proj.load_state_dict(cvg.weights(image_proj, "proj"), strict=False)
    image_prompt_embeds = image_proj(clip_image_embeds)
    uncond_image_prompt_embeds = image_proj(torch.zeros_like(clip_image_embeds))
    assert image_prompt_embeds.dtype == torch.float16 and image_prompt_embeds.shape == (cvg.BATCH, 4, 768)
    e_tok = rel(image_prompt_embeds, ref["tokens"])
    e_un = rel(uncond_image_prompt_embeds, ref["uncond_tokens"])
    print(f"fp16 parameters: image_embeds {e_emb:.3e}, text_embeds {e_txt:.3e}, tokens {e_tok:.3e}, uncond {e_un:.3e}")
    assert e_emb < TOL16["image_embeds"] and e_txt < TOL16["text_embeds"]
    assert e_tok < TOL16["tokens"] and e_un < TOL16["uncond"]
    # the negative content prompt subtraction runs in fp16 as in the app
    emb = clip_image_embeds - 0.5 * neg_content_emb
    assert torch.isfinite(image_proj(emb)).all()


def test_weight_reload_changes_the_output():
    model = vision("tiny")
    px = cvg.pixels(cvg.BATCH).cuda()
    e0 = model(px).image_embeds
    model.load_state_dict(cvg.weights(model, "vision", seed=1))
    e1 = model(px).image_embeds
    assert rel(e0, e1) > 0.1
    assert torch.equal(e1, vision("tiny", seed=1)(px).image_embeds)


# ------------------------------------------------------------------------------------------------ style sampling
def test_style_sampling_with_our_image_prompt(g):
    """DDIM on the tiny style model with c_ip from our encoder and projection (the app's :389-409 with swapped imports)
    against the same call with c_ip from transformers and the reference's ImageProjModel (the fixture's tokens)"""
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from cldm.ddim_hacked import DDIMSampler
    from oracle import synth
    gold = os.path.join(ROOT, "tests", "golden")
    sg = torch.load(os.path.join(gold, "tiny_style_golden.pt"), weights_only=False)
    m = create_model(os.path.join(gold, "tiny_style.yaml"), init_weights=False)
    m.control_model.load_state_dict(synth.synth_state_dict(sg["control_shapes"], sg["seed"], "control_model."), strict=True)
    m.model.diffusion_model.load_state_dict(synth.synth_state_dict(sg["unet_shapes"], sg["seed"], "model.diffusion_model."),
                                            strict=True)
    model = m.cuda().eval()
    B, H = cvg.BATCH, sg["H"]
    hint = synth.synth_input("hint", (B, 4, H, H), 7).cuda()
    ctx = synth.synth_input("ctx", (B, 77, 64), 7).cuda()
    x_T = synth.synth_input("x", (B, 4, H, H), 7).cuda()

    enc, proj = vision("tiny"), image_proj("tiny")
    emb = enc(cvg.pixels(B).cuda()).image_embeds
    ours = (proj(emb), proj(torch.zeros_like(emb)))
    theirs = (g["vision_tiny"]["tokens"].cuda(), g["vision_tiny"]["uncond_tokens"].cuda())

    def sample(ip, uip):
        sampler = DDIMSampler(model)
        out, _ = sampler.sample(4, B, (4, H, H), conditioning={"c_concat": [hint], "c_crossattn": [ctx], "c_ip": [ip]},
                                verbose=False, x_T=x_T.clone(), eta=0.0, unconditional_guidance_scale=7.5,
                                unconditional_conditioning={"c_concat": [hint], "c_crossattn": [ctx], "c_ip": [uip]})
        torch.cuda.synchronize()
        return out

    a, b = sample(*ours), sample(*theirs)
    err = rel(a, b)
    print(f"style DDIM sample, our c_ip vs the fixture's: rel err {err:.3e}")
    assert torch.isfinite(a).all() and err < SAMPLE_TOL
    assert torch.equal(sample(*ours), a)
