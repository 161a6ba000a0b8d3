"""The CLIP text encoder on the sm_90a kernels: the causal attention kernel against fp32 torch, the tiny and SD1.5-size
encoders against the reference's FrozenCLIPEmbedder (tests/golden/clip_text_golden.pt, `tools/make_clip_golden.py`) and
against transformers' CLIPTextModel on the same weights, prompts through an opted-in model's conditioning and DDIM
sampling, weight reloads, and checkpoints.  Errors are printed under `pytest -s`."""
import ctypes as C
import os

import pytest
import torch

import clip_golden

pytestmark = pytest.mark.gpu
ROOT = clip_golden.ROOT
TINY_YAML = os.path.join(ROOT, "tests", "golden", "tiny_finetune.yaml")

# Norm-relative error bounds (||z - ref|| / ||ref||), about 20 % above what an H100 measured (printed with -s).  The
# reference is fp32 throughout; here the GEMM operands and the attention are fp16 with fp32 accumulation, the residual
# stream and LayerNorm statistics fp32.
TOL = {
    # measured against the reference's fixture / against transformers on a ragged batch
    ("tiny", "last"): 7.3e-4,       # 6.07e-4 / 6.05e-4
    ("tiny", "hidden-2"): 7.1e-4,   # 5.90e-4 / 5.84e-4
    ("tiny", "pooled"): 7.1e-4,     # 5.51e-4 / 5.91e-4
    ("sd15", "last"): 8.9e-4,       # 7.40e-4 / 7.30e-4
    ("sd15", "hidden-2"): 8.6e-4,   # 7.17e-4 / 7.14e-4
    ("sd15", "pooled"): 1.01e-3,    # 8.27e-4 / 8.42e-4
}
ATTN_TOL = 4.2e-4  # max |err| / max |ref| of the causal kernel (fp16 P and V): 3.43e-4 measured at n = 128
LAYERS = {"last": {}, "hidden-2": {"layer": "hidden", "layer_idx": -2}, "pooled": {"layer": "pooled"}}


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(scope="module")
def g():
    return clip_golden.load()


@pytest.fixture(scope="module")
def dirs(g, tmp_path_factory):
    base = tmp_path_factory.mktemp("clip")
    return {w: clip_golden.write_version_dir(str(base / w), g, w) for w in ("tiny", "sd15")}


def encoder(path, seed=clip_golden.SEED, **kw):
    from ctrlora_b200.text_encoder import FrozenCLIPEmbedder
    enc = FrozenCLIPEmbedder(version=path, **kw)
    enc.load_state_dict(clip_golden.embedder_weights(enc, seed), strict=True)
    return enc.cuda()


# ------------------------------------------------------------------------------------------------ the causal kernel
@pytest.mark.parametrize("batch", [1, 16])
@pytest.mark.parametrize("n", [1, 7, 64, 77, 128])
def test_causal_attention(n, batch):
    from ctrlora_b200 import ops
    heads, d = 12, 64
    gen = torch.Generator(device="cuda").manual_seed(n * 100 + batch)
    q, k, v = (torch.randn((batch, n, heads * d), device="cuda", generator=gen).half() for _ in range(3))
    n_pad = (n + 7) // 8 * 8 + 8
    vt = torch.full((batch, heads, d, n_pad), float("nan"), device="cuda", dtype=torch.float16)  # padding is never read
    vt[..., :n] = v.view(batch, n, heads, d).permute(0, 2, 3, 1)
    rows = batch * n
    buf = torch.full((rows + 16, heads * d), 7.0, device="cuda", dtype=torch.float16)
    out = ops.causal_attention(q.view(rows, -1), k.view(rows, -1), vt, batch, heads, n, out=buf[:rows])
    again = ops.causal_attention(q.view(rows, -1), k.view(rows, -1), vt, batch, heads, n)
    torch.cuda.synchronize()
    assert torch.equal(out, again)
    assert (buf[rows:] == 7.0).all()  # nothing beyond the last row is stored
    qf, kf, vf = (t.float().view(batch, n, heads, d).transpose(1, 2) for t in (q, k, v))
    s = qf @ kf.transpose(-1, -2) / 8.0
    s = s.masked_fill(torch.ones(n, n, device="cuda", dtype=torch.bool).triu(1), float("-inf"))
    ref = (s.softmax(-1) @ vf).transpose(1, 2).reshape(rows, heads * d)
    err = ((out.float() - ref).abs().max() / ref.abs().max()).item()
    print(f"causal attention n={n} batch={batch}: max err {err:.2e}")
    assert err < ATTN_TOL


def test_causal_attention_unsupported():
    from ctrlora_b200 import _lib, ops
    t = torch.zeros((129, 64), device="cuda", dtype=torch.float16)
    vt = torch.zeros((1, 1, 64, 136), device="cuda", dtype=torch.float16)
    with pytest.raises(_lib.CtrloraError, match="unsupported"):
        ops.causal_attention(t, t, vt, 1, 1, 129)
    lib = _lib.load()
    t80 = torch.zeros((8, 80), device="cuda", dtype=torch.float16)
    st = lib.ctrlora_causal_attention_f16(t80.data_ptr(), 80, t80.data_ptr(), 80, vt.data_ptr(), 8, t80.data_ptr(), 80, 1, 1,
                                          8, 80, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 4  # CTRLORA_STATUS_UNSUPPORTED


# ------------------------------------------------------------------------------------------------ the encoder
@pytest.mark.parametrize("which", ["tiny", "sd15"])
def test_encoder_against_reference(g, dirs, which):
    ref = g[which]
    for name, kw in LAYERS.items():
        enc = encoder(dirs[which], **kw)
        z = enc.encode_tokens(ref["ids"])
        assert z.dtype == torch.float32 and z.is_cuda and z.shape == ref[name].shape
        err = rel(z, ref[name])
        enc.residual_f32 = False
        err16 = rel(enc.encode_tokens(ref["ids"]), ref[name])
        enc.residual_f32 = True
        print(f"{which} {name}: rel err {err:.3e} (fp16 residual stream: {err16:.3e})")
        assert err < TOL[(which, name)], (which, name, err)
        # strings go through the reference's tokenizer call to the same ids and the same bits
        assert torch.equal(enc.encode(g["prompts"]), z)
        assert torch.equal(enc.encode_tokens(ref["ids"].cuda()), z)
        del enc


RAGGED = ["a cat", "the photo of the cat on the mat", "", "of the photo of the cat of the mat of the photo of the cat of the "
          "mat of the photo of the cat of the mat", "x"]


@pytest.mark.parametrize("which", ["tiny", "sd15"])
def test_encoder_against_transformers(g, dirs, which):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = g[which]["config"]
    hf = CLIPTextModel(CLIPTextConfig(**cfg)).eval()
    shapes = {k: tuple(v.shape) for k, v in hf.state_dict().items()}
    hf.load_state_dict(clip_golden.synth_text_weights(shapes), strict=True)
    hf = hf.cuda()
    for name, kw in LAYERS.items():
        enc = encoder(dirs[which], **kw)
        ids = enc.tokenize(RAGGED)
        with torch.no_grad():
            out = hf(input_ids=ids.cuda(), output_hidden_states=True)
        ref = {"last": out.last_hidden_state, "hidden-2": out.hidden_states[-2], "pooled": out.pooler_output[:, None]}[name]
        err = rel(enc.encode_tokens(ids), ref)
        print(f"{which} {name} vs transformers, ragged batch of {len(RAGGED)}: rel err {err:.3e}")
        assert err < TOL[(which, name)], (which, name, err)
        del enc


def test_weights_reload_invalidates_kernel_copies(g, dirs):
    enc = encoder(dirs["tiny"])
    ids = g["tiny"]["ids"]
    z0 = enc.encode_tokens(ids)
    enc.load_state_dict(clip_golden.embedder_weights(enc, seed=1))
    z1 = enc.encode_tokens(ids)
    fresh = encoder(dirs["tiny"], seed=1).encode_tokens(ids)
    assert rel(z0, z1) > 0.1
    assert torch.equal(z1, fresh)


# ------------------------------------------------------------------------------------------------ an opted-in model
def _tiny_model(dirs, seed=7, text_encoder=True):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    from oracle import synth
    te = {"version": dirs["tiny"]} if text_encoder else False
    model = create_model(TINY_YAML, init_weights=False, text_encoder=te)
    for sub, prefix in ((model.control_model, "control_model."), (model.model.diffusion_model, "model.diffusion_model.")):
        shapes = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
        sub.load_state_dict(synth.synth_state_dict(shapes, seed, prefix))
    if text_encoder:
        model.cond_stage_model.load_state_dict(clip_golden.embedder_weights(model.cond_stage_model))
    return model.cuda().eval()


def test_conditioning_and_sampling_from_prompts(g, dirs):
    model = _tiny_model(dirs)
    from cldm.ddim_hacked import DDIMSampler
    from oracle import synth
    enc = model.cond_stage_model
    prompts = g["prompts"]
    c = model.get_learned_conditioning(prompts)
    ids = g["tiny"]["ids"]
    c_ids = enc.encode_tokens(ids)
    assert c.shape == (3, 77, 64) and torch.equal(c, c_ids)
    assert rel(c, g["tiny"]["last"]) < TOL[("tiny", "last")]
    uc = model.get_unconditional_conditioning(3)
    assert torch.equal(uc, enc.encode_tokens(enc.tokenize([""] * 3)))
    B, H = 3, 16
    hint = synth.synth_input("hint", (B, 4, H, H), 7).cuda()
    x_T = synth.synth_input("x", (B, 4, H, H), 7).cuda()

    def sample(ctx, uctx):
        sampler = DDIMSampler(model)
        out, _ = sampler.sample(4, B, (4, H, H), conditioning={"c_concat": [hint], "c_crossattn": [ctx]}, verbose=False,
                                x_T=x_T.clone(), eta=0.0, unconditional_guidance_scale=7.5,
                                unconditional_conditioning={"c_concat": [hint], "c_crossattn": [uctx]})
        torch.cuda.synchronize()
        return out

    a = sample(model.get_learned_conditioning(prompts), model.get_unconditional_conditioning(B))
    b = sample(enc.encode_tokens(ids), enc.encode_tokens(enc.tokenize([""] * B)))
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)


def test_checkpoint_round_trip(g, dirs, tmp_path):
    from ctrlora_b200.train import FinetuneTrainer
    model = _tiny_model(dirs)
    path = str(tmp_path / "opted.ckpt")
    FinetuneTrainer(model, lr=1e-5).save_checkpoint(path)
    sd = torch.load(path, map_location="cpu", weights_only=True)["state_dict"]
    assert [k for k in sd if k.startswith("cond_stage_model.")] == [
        "cond_stage_model." + k for k in model.cond_stage_model.state_dict()]
    ids = g["tiny"]["ids"]
    z = model.cond_stage_model.encode_tokens(ids)

    other = _tiny_model(dirs)
    other.cond_stage_model.load_state_dict(clip_golden.embedder_weights(other.cond_stage_model, seed=3))
    assert not torch.equal(other.cond_stage_model.encode_tokens(ids), z)
    FinetuneTrainer(other, lr=1e-5).load_checkpoint(path)
    assert torch.equal(other.cond_stage_model.encode_tokens(ids), z)

    # a model that did not opt in ignores the file's CLIP weights
    plain = _tiny_model(dirs, text_encoder=False)
    assert plain.cond_stage_model is None
    FinetuneTrainer(plain, lr=1e-5).load_checkpoint(path)
    assert not any(k.startswith("cond_stage_model.") for k in plain.state_dict())
