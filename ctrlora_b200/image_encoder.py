"""The style app's image-prompt models on the sm_90a kernels (app/gradio_ctrlora_style_transfer.py:385-409):

- `CLIPVisionModelWithProjection`: transformers' class of that name, the IP-Adapter's CLIP ViT-H/14 image encoder, which
  turns the preprocessed style image into `image_embeds`;
- `ImageProjModel`: the app's projection (:93-111), `image_embeds` -> 4 image-prompt tokens `c_ip`;
- `CLIPTextModelWithProjection`: transformers' class of that name, the ViT-H text tower whose `text_embeds` the app
  subtracts from the image embedding when "negative content prompt" is on.

Switching the app over is an import swap; `CLIPImageProcessor` and `CLIPTokenizer` stay transformers' host-side code.
The modules keep transformers' state-dict keys and the app's calls (`from_pretrained(dir).to('cuda', dtype=torch.float16)`,
`model(pixel_values).image_embeds`, `model(**tokens).text_embeds`).  Nothing is fetched: `from_pretrained` reads a local
directory and nothing else.

The vision forward: a patch gather plus one ctrlora_gemm_f16 for the patch Conv2d, the class + position embedding
assembly, pre_layrnorm, the CLIP layer loop of text_encoder.run_layers with the full-attention kernel (d_head 80 at
ViT-H) and exact GELU, post_layernorm on the class rows and visual_projection.  The residual stream is fp32, GEMM operands
fp16 with fp32 accumulation.  Parameters may be fp32 or fp16: the kernels read fp16 GEMM copies and fp32 LayerNorm
parameters, biases and embeddings from a PrepCache (so load_state_dict invalidates them), and the outputs take the
parameters' dtype, as transformers' do.  Inference only: no autograd, on the current stream.
"""
import json
import os

import torch
import torch.nn as nn

from . import ops, prepare
from .text_encoder import _Encoder, _TextModel, check_text_config, pooled_rows, run_layers

# the IP-Adapter SD1.5 image_encoder (CLIP ViT-H/14, laion2B): its config.json
VIT_H_VISION_CONFIG = {"hidden_size": 1280, "intermediate_size": 5120, "num_hidden_layers": 32, "num_attention_heads": 16,
                       "num_channels": 3, "image_size": 224, "patch_size": 14, "projection_dim": 1024, "hidden_act": "gelu",
                       "layer_norm_eps": 1e-5}
# the text tower of the same CLIP (laion/CLIP-ViT-H-14-laion2B-s32B-b79K's "text_config"; eos_token_id 2 there, so the
# pooled row is the argmax token id)
VIT_H_TEXT_CONFIG = {"vocab_size": 49408, "hidden_size": 1024, "intermediate_size": 4096, "num_hidden_layers": 24,
                     "num_attention_heads": 16, "max_position_embeddings": 77, "hidden_act": "gelu", "layer_norm_eps": 1e-5,
                     "projection_dim": 1024, "eos_token_id": 2}
ACTS = ("gelu", "quick_gelu")


class ModelOutput(dict):
    """transformers-style output: fields by attribute, by name or by position"""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e

    def __getitem__(self, key):
        if isinstance(key, int):
            return list(self.values())[key]
        return super().__getitem__(key)


def _config(config, defaults, sub):
    """defaults updated by `config` (a dict, a transformers config object, or None); a CLIPConfig's `sub` entry is used"""
    cfg = dict(defaults)
    if config is not None:
        raw = config if isinstance(config, dict) else config.to_dict()
        raw = raw.get(sub) or raw
        cfg.update({k: raw[k] for k in cfg if k in raw})
    return cfg


def vision_config(config=None):
    """the vision-tower architecture: the built-in ViT-H/14 updated by `config`; ValueError if the kernels cannot run it"""
    cfg = _config(config, VIT_H_VISION_CONFIG, "vision_config")
    c, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    if cfg["hidden_act"] not in ACTS:
        raise ValueError(f"CLIP vision config: hidden_act {cfg['hidden_act']!r}, only {' / '.join(ACTS)} is implemented")
    if c % heads or (c // heads) % 8 or c // heads > 160:
        raise ValueError(f"CLIP vision config: head size {c} / {heads}, the attention kernel takes a multiple of 8 up to 160")
    if c > 2048 or cfg["intermediate_size"] % 8:
        raise ValueError(f"CLIP vision config: hidden {c} / MLP {cfg['intermediate_size']}, at most 2048 and a multiple "
                         "of 8 are supported")
    if cfg["image_size"] % cfg["patch_size"]:
        raise ValueError(f"CLIP vision config: image size {cfg['image_size']} is not a multiple of the patch size "
                         f"{cfg['patch_size']}")
    return cfg


def text_config(config=None):
    """the text-tower architecture: the built-in ViT-H/14 text tower updated by `config`"""
    cfg = _config(config, VIT_H_TEXT_CONFIG, "text_config")
    check_text_config(cfg, "CLIPTextModelWithProjection", ACTS)
    return cfg


def _local_config(path):
    if not os.path.isdir(str(path)):
        raise OSError(f"{path!r} is not a local directory: ctrlora_b200 loads CLIP weights from a directory with "
                      "config.json and model.safetensors or pytorch_model.bin, and never downloads them")
    cfg_path = os.path.join(str(path), "config.json")
    if not os.path.isfile(cfg_path):
        raise OSError(f"no config.json in {path!r}")
    with open(cfg_path) as f:
        return json.load(f)


def _local_weights(path, prefixes):
    """the state dict in `path` (model.safetensors, its sharded index, or pytorch_model.bin), restricted to the keys
    under `prefixes`: a full CLIPModel checkpoint holds both towers, and each model takes its own"""
    path = str(path)
    st, idx, pt = (os.path.join(path, f) for f in ("model.safetensors", "model.safetensors.index.json", "pytorch_model.bin"))
    if os.path.isfile(st) or os.path.isfile(idx):
        from safetensors.torch import load_file
        if os.path.isfile(st):
            files = [st]
        else:
            with open(idx) as f:
                files = [os.path.join(path, n) for n in sorted(set(json.load(f)["weight_map"].values()))]
        sd = {}
        for fn in files:
            sd.update(load_file(fn))
    elif os.path.isfile(pt):
        sd = torch.load(pt, map_location="cpu", weights_only=True)
    else:
        raise OSError(f"no model.safetensors or pytorch_model.bin in {path!r}")
    return {k: v for k, v in sd.items() if k.startswith(prefixes)}


class _Frozen(nn.Module):
    """inference-only module: parameters frozen, eval mode, fp16/fp32 kernel copies in a PrepCache"""

    def _setup(self):
        self.eval()
        for p in self.parameters():
            p.requires_grad = False
        self.__dict__["_prep"] = prepare.PrepCache()

    def _device(self, p):
        if p.device.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} runs on the sm_90a kernels only: move the model to a CUDA device")
        return p.device

    def _f32(self, key, p):
        return self._prep.get(key, [p], lambda: prepare.bias_f32(p))

    def _ln(self, key, ln):
        return self._prep.get(key, [ln.weight, ln.bias], lambda: (prepare.bias_f32(ln.weight), prepare.bias_f32(ln.bias), ln.eps))

    def _proj(self, key, lin):
        """fp16 [N, K] weight and fp32 bias (or None) for ctrlora_small_linear"""
        def build():
            n, k = lin.weight.shape
            return prepare.linear_weight(lin.weight).view(n, k), prepare.bias_f32(lin.bias)
        return self._prep.get(key, [lin.weight, lin.bias], build)


# ------------------------------------------------------------------------------------------------ vision tower
class _VisionEmbeddings(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        c, p = cfg["hidden_size"], cfg["patch_size"]
        self.class_embedding = nn.Parameter(torch.zeros(c))
        self.patch_embedding = nn.Conv2d(cfg["num_channels"], c, kernel_size=p, stride=p, bias=False)
        self.position_embedding = nn.Embedding((cfg["image_size"] // p) ** 2 + 1, c)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # checkpoints written by transformers 4 carry the position_ids buffer; it is always arange(P + 1)
        state_dict.pop(prefix + "position_ids", None)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


class _VisionTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        c, eps = cfg["hidden_size"], cfg["layer_norm_eps"]
        self.embeddings = _VisionEmbeddings(cfg)
        self.pre_layrnorm = nn.LayerNorm(c, eps=eps)  # transformers' spelling
        self.encoder = _Encoder(cfg)
        self.post_layernorm = nn.LayerNorm(c, eps=eps)


class CLIPVisionModelWithProjection(_Frozen):
    """transformers' CLIPVisionModelWithProjection (keys vision_model.*, visual_projection.weight) on the sm_90a kernels.
    forward(pixel_values [B, C, S, S]) -> .image_embeds [B, projection_dim], .last_hidden_state [B, P + 1, hidden]."""

    def __init__(self, config=None):
        super().__init__()
        self.config = vision_config(config)
        self.vision_model = _VisionTransformer(self.config)
        self.visual_projection = nn.Linear(self.config["hidden_size"], self.config["projection_dim"], bias=False)
        self._setup()

    @classmethod
    def from_pretrained(cls, path, **kwargs):
        """config.json (a CLIPVisionConfig, or a CLIPConfig with vision_config) and the weights of a local directory.
        Loading options of transformers' from_pretrained (torch_dtype, ...) are not taken: use .to() afterwards."""
        model = cls(_local_config(path))
        model.load_state_dict(_local_weights(path, ("vision_model.", "visual_projection.")), strict=True)
        return model

    def _patch_weight(self):
        """the patch Conv2d as a GEMM weight: fp16 [C, 1, k_pad], columns in (c, kh, kw) order, zero beyond K"""
        conv = self.vision_model.embeddings.patch_embedding

        def build():
            c = conv.weight.shape[0]
            k = conv.weight[0].numel()
            w = torch.zeros((c, 1, (k + 7) // 8 * 8), device=conv.weight.device, dtype=torch.float16)
            w[:, :, :k] = prepare.linear_weight(conv.weight.detach().reshape(c, k))
            return w
        return self._prep.get("patch", [conv.weight], build)

    @torch.no_grad()
    def forward(self, pixel_values, output_attentions=None, output_hidden_states=None, return_dict=None, **kwargs):
        if output_hidden_states:
            raise NotImplementedError("output_hidden_states (IP-Adapter-Plus' penultimate layer) is not implemented")
        if output_attentions:
            raise NotImplementedError("output_attentions is not implemented")
        vm, cfg = self.vision_model, self.config
        emb = vm.embeddings
        dev = self._device(emb.class_embedding)
        s, p, c = cfg["image_size"], cfg["patch_size"], cfg["hidden_size"]
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (cfg["num_channels"], s, s):
            raise ValueError(f"pixel_values must be [B, {cfg['num_channels']}, {s}, {s}], got {tuple(pixel_values.shape)}")
        px = pixel_values.to(dev)
        if px.dtype not in (torch.float32, torch.float16):
            px = px.float()
        px = px.contiguous()
        b = px.shape[0]
        patches = (s // p) ** 2
        w_patch = self._patch_weight()
        rows = ops.clip_patch_gather(px, p, w_patch.shape[-1])
        patch_out = ops.gemm(rows, w_patch, out_f32=True)
        h = ops.clip_vision_embed(patch_out, self._f32("cls", emb.class_embedding),
                                  self._f32("pos", emb.position_embedding.weight), b)
        h = ops.layernorm_rows(h, *self._ln("pre_ln", vm.pre_layrnorm), out_f32=True)
        h = run_layers(vm.encoder.layers, self._prep, h, b, patches + 1, cfg["num_attention_heads"], cfg["hidden_act"],
                       causal=False)
        pooled = ops.layernorm_rows(h.view(b, patches + 1, c)[:, 0], *self._ln("post_ln", vm.post_layernorm), out_f32=True)
        w_proj, _ = self._proj("proj", self.visual_projection)
        image_embeds = ops.small_linear(pooled, w_proj, None)
        dt = self.visual_projection.weight.dtype
        return ModelOutput(image_embeds=image_embeds.to(dt), last_hidden_state=h.view(b, patches + 1, c).to(dt))


# ------------------------------------------------------------------------------------------------ image prompt tokens
class ImageProjModel(_Frozen):
    """Projection Model (app/gradio_ctrlora_style_transfer.py:93-111): image_embeds [B, clip_embeddings_dim] ->
    LayerNorm(proj(image_embeds)) as [B, clip_extra_context_tokens, cross_attention_dim], on the kernels."""

    def __init__(self, cross_attention_dim=768, clip_embeddings_dim=1024, clip_extra_context_tokens=4):
        super().__init__()
        self.generator = None
        self.cross_attention_dim = cross_attention_dim
        self.clip_extra_context_tokens = clip_extra_context_tokens
        self.proj = torch.nn.Linear(clip_embeddings_dim, self.clip_extra_context_tokens * cross_attention_dim)
        self.norm = torch.nn.LayerNorm(cross_attention_dim)
        self._setup()

    @torch.no_grad()
    def forward(self, image_embeds):
        dev = self._device(self.proj.weight)
        x = image_embeds.to(dev).reshape(-1, self.proj.in_features)
        x = x.float().contiguous()
        w, bias = self._proj("proj", self.proj)
        y = ops.small_linear(x, w, bias)
        out = ops.layernorm_rows(y.view(-1, self.cross_attention_dim), *self._ln("norm", self.norm), out_f32=True)
        return out.view(-1, self.clip_extra_context_tokens, self.cross_attention_dim).to(self.proj.weight.dtype)


# ------------------------------------------------------------------------------------------------ text tower
class CLIPTextModelWithProjection(_Frozen):
    """transformers' CLIPTextModelWithProjection (keys text_model.*, text_projection.weight) on the sm_90a kernels.
    forward(input_ids [B, n], attention_mask=None) -> .text_embeds [B, projection_dim] (the projected final-LayerNorm
    row of each sequence's EOS token), .last_hidden_state [B, n, hidden].  A right-padded attention_mask (ones, then
    zeros) is accepted: under the causal mask no padded key reaches a row before it, so text_embeds and the rows of the
    real tokens are transformers'; the padded rows themselves are not."""

    def __init__(self, config=None):
        super().__init__()
        self.config = text_config(config)
        self.text_model = _TextModel(self.config)
        self.text_projection = nn.Linear(self.config["hidden_size"], self.config["projection_dim"], bias=False)
        self._setup()

    @classmethod
    def from_pretrained(cls, path, **kwargs):
        """config.json (a CLIPTextConfig, or a CLIPConfig with text_config) and the weights of a local directory"""
        model = cls(_local_config(path))
        model.load_state_dict(_local_weights(path, ("text_model.", "text_projection.")), strict=True)
        return model

    @torch.no_grad()
    def forward(self, input_ids, attention_mask=None, position_ids=None, output_attentions=None, output_hidden_states=None,
                return_dict=None, **kwargs):
        if output_hidden_states or output_attentions:
            raise NotImplementedError("output_hidden_states / output_attentions are not implemented")
        if position_ids is not None:
            raise NotImplementedError("position_ids other than the default arange(n) are not implemented")
        tm, cfg = self.text_model, self.config
        if input_ids.dtype != torch.int64 or input_ids.dim() != 2:
            raise ValueError(f"input_ids must be int64 [B, n], got {input_ids.dtype} {tuple(input_ids.shape)}")
        b, n = input_ids.shape
        if n > cfg["max_position_embeddings"]:
            raise ValueError(f"{n} tokens, the model has {cfg['max_position_embeddings']} positions")
        if attention_mask is not None:
            m = attention_mask.detach().cpu()
            if (m.shape != input_ids.shape or not ((m == 0) | (m == 1)).all() or (b and not (m[:, 0] == 1).all())
                    or not (m[:, 1:] <= m[:, :-1]).all()):
                raise ValueError("attention_mask must be right padding: per row ones, then zeros (at least one 1)")
        dev = self._device(tm.embeddings.token_embedding.weight)
        ids = input_ids.to(dev).contiguous()
        emb = tm.embeddings
        h = ops.clip_embed(ids, self._f32("tok", emb.token_embedding.weight), self._f32("pos", emb.position_embedding.weight))
        h = run_layers(tm.encoder.layers, self._prep, h, b, n, cfg["num_attention_heads"], cfg["hidden_act"], causal=True)
        h = ops.layernorm_rows(h, *self._ln("final_ln", tm.final_layer_norm), out_f32=True)
        z = h.view(b, n, -1)
        pooled = z[torch.arange(b, device=dev), pooled_rows(ids, cfg["eos_token_id"])].contiguous()
        w_proj, _ = self._proj("proj", self.text_projection)
        text_embeds = ops.small_linear(pooled, w_proj, None)
        dt = self.text_projection.weight.dtype
        return ModelOutput(text_embeds=text_embeds.to(dt), last_hidden_state=z.to(dt))
