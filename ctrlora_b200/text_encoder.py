"""The reference's CLIP text encoder on the sm_90a kernels: `FrozenCLIPEmbedder` (ldm/modules/encoders/modules.py:88-135),
which tokenizes prompts and runs transformers' `CLIPTextModel` (openai/clip-vit-large-patch14 for SD1.5).

The module keeps the reference's signature, `LAYERS`, asserts and state-dict keys (`transformer.text_model.*`), so an
SD1.5 checkpoint's `cond_stage_model.*` weights load into it with `model.load_state_dict(sd, strict=False)`.  Nothing is
fetched: the architecture is built in (or read from `version/config.json` when `version` is a local directory), the
weights come from the checkpoint, and the tokenizer is built on the first call that passes strings.

Per layer the forward is four ctrlora_gemm_f16 launches (one stacked q|k|v GEMM that stores V transposed, out_proj +
residual, fc1, fc2 + residual), ctrlora_causal_attention_f16, ctrlora_quick_gelu_f16 and two ctrlora_layernorm_rows.
That layer loop (`run_layers`) is shared with the image-prompt towers of `image_encoder.py`, which add exact GELU and
full (non-causal) attention.  The residual stream stays fp32 like the reference's (CLIP-L's activations carry large outliers at the EOS position,
which an fp16 stream rounds coarsely; DESIGN.md §3 has the measured errors of both).
It is inference only: no autograd, parameters frozen.
"""
import json
import os

import torch
import torch.nn as nn

from . import ops, prepare

# openai/clip-vit-large-patch14's text tower (its config.json "text_config"; eos_token_id 2 there, so the pooled row is
# the argmax token id, see _pooled_rows)
CLIP_L_CONFIG = {"vocab_size": 49408, "hidden_size": 768, "intermediate_size": 3072, "num_hidden_layers": 12,
                 "num_attention_heads": 12, "max_position_embeddings": 77, "hidden_act": "quick_gelu",
                 "layer_norm_eps": 1e-5, "eos_token_id": 2}


def text_config(version):
    """The text-tower architecture for `version`: a local directory's config.json (a CLIPTextConfig, or a CLIPConfig
    with a "text_config" entry), else the built-in CLIP ViT-L/14 one.  Never touches the network."""
    cfg = dict(CLIP_L_CONFIG)
    path = os.path.join(str(version), "config.json")
    if os.path.isdir(str(version)) and os.path.isfile(path):
        with open(path) as f:
            raw = json.load(f)
        raw = raw.get("text_config", raw)
        cfg.update({k: raw[k] for k in cfg if k in raw})
    check_text_config(cfg, version, ("quick_gelu",))
    return cfg


def check_text_config(cfg, version, acts):
    """raise ValueError unless the causal d_head-64 layer loop runs `cfg` (hidden_act one of `acts`)"""
    if cfg["hidden_act"] not in acts:
        raise ValueError(f"CLIP text config of {version!r}: hidden_act {cfg['hidden_act']!r}, only "
                         f"{' / '.join(acts)} is implemented")
    if cfg["hidden_size"] != 64 * cfg["num_attention_heads"]:
        raise ValueError(f"CLIP text config of {version!r}: head size {cfg['hidden_size']} / {cfg['num_attention_heads']}, "
                         "the causal attention kernel takes 64")
    if cfg["max_position_embeddings"] > 128:
        raise ValueError(f"CLIP text config of {version!r}: {cfg['max_position_embeddings']} positions, at most 128 are "
                         "supported")


class _Embeddings(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.token_embedding = nn.Embedding(cfg["vocab_size"], cfg["hidden_size"])
        self.position_embedding = nn.Embedding(cfg["max_position_embeddings"], cfg["hidden_size"])

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # SD1.5 files carry the position_ids buffer that transformers 4 persisted; it is always arange(77)
        state_dict.pop(prefix + "position_ids", None)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


class _Attention(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(c, c) for _ in range(4))


class _MLP(nn.Module):
    def __init__(self, c, inner):
        super().__init__()
        self.fc1 = nn.Linear(c, inner)
        self.fc2 = nn.Linear(inner, c)


class _Layer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        c = cfg["hidden_size"]
        self.self_attn = _Attention(c)
        self.layer_norm1 = nn.LayerNorm(c, eps=cfg["layer_norm_eps"])
        self.mlp = _MLP(c, cfg["intermediate_size"])
        self.layer_norm2 = nn.LayerNorm(c, eps=cfg["layer_norm_eps"])


class _Encoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.layers = nn.ModuleList(_Layer(cfg) for _ in range(cfg["num_hidden_layers"]))


class _TextModel(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = _Embeddings(cfg)
        self.encoder = _Encoder(cfg)
        self.final_layer_norm = nn.LayerNorm(cfg["hidden_size"], eps=cfg["layer_norm_eps"])


class _Transformer(nn.Module):
    """holds `text_model` so the keys are CLIPTextModel's: transformer.text_model.*"""

    def __init__(self, cfg):
        super().__init__()
        self.text_model = _TextModel(cfg)


def pooled_rows(ids, eos):
    """the EOS row of each sequence, as transformers' CLIPTextTransformer picks it: the largest token id when the
    config's eos_token_id is 2 (the original CLIP configs), else the first occurrence of eos_token_id"""
    if eos == 2:
        return ids.to(torch.int).argmax(dim=-1)
    return (ids.to(torch.int) == eos).int().argmax(dim=-1)


def layer_weights(prep, layer, i):
    """kernel copies of CLIP encoder layer i from `prep` (a PrepCache): fp16 stacked q|k|v [3C, 1, C] + fp32 bias,
    out_proj, fc1 and fc2 as (fp16 [N, 1, K], fp32 bias), and layer_norm1 / layer_norm2 as fp32 (gamma, beta, eps).
    fp32 parameters are used as they are; fp16 ones (a module moved with .to(dtype=torch.float16)) get fp32 copies."""
    at, mlp = layer.self_attn, layer.mlp
    lins = (at.q_proj, at.k_proj, at.v_proj)

    def qkv():
        c = at.q_proj.in_features
        w = torch.empty((3 * c, 1, c), device=at.q_proj.weight.device, dtype=torch.float16)
        for j, lin in enumerate(lins):
            prepare.linear_weight(lin.weight, out=w[j * c:(j + 1) * c])
        return w, torch.cat([prepare.bias_f32(lin.bias) for lin in lins])

    def lin(m):
        return lambda: (prepare.linear_weight(m.weight), prepare.bias_f32(m.bias))

    def ln(m):
        return lambda: (prepare.bias_f32(m.weight), prepare.bias_f32(m.bias), m.eps)

    get = prep.get
    return (get(("qkv", i), [p for m in lins for p in (m.weight, m.bias)], qkv),
            get(("out", i), [at.out_proj.weight, at.out_proj.bias], lin(at.out_proj)),
            get(("fc1", i), [mlp.fc1.weight, mlp.fc1.bias], lin(mlp.fc1)),
            get(("fc2", i), [mlp.fc2.weight, mlp.fc2.bias], lin(mlp.fc2)),
            get(("ln1", i), [layer.layer_norm1.weight, layer.layer_norm1.bias], ln(layer.layer_norm1)),
            get(("ln2", i), [layer.layer_norm2.weight, layer.layer_norm2.bias], ln(layer.layer_norm2)))


def run_layers(layers, prep, h, b, n, heads, hidden_act, causal, f32=True, weights=layer_weights, keep=(), split_k=0):
    """CLIPEncoder over `layers` on the residual stream h ([b * n, C], fp32 when f32, else fp16): per layer
    layer_norm1, one stacked q|k|v GEMM that stores V transposed, self-attention (causal d_head 64, or the full
    ctrlora_attention_f16), out_proj + residual, layer_norm2, fc1, GELU (hidden_act "quick_gelu" or "gelu", in place),
    fc2 + residual.  Returns the new residual stream.
    weights(prep, layer, i): layer i's kernel copies in layer_weights' form (default: CLIP's parameter names).
    keep: layer indices after which the stream is handed back; when given, returns (h, [h after each kept layer]).
    split_k: passed to every GEMM (0 lets the tile model choose)."""
    kept = []
    dev = h.device
    c = h.shape[1]
    d = c // heads
    n_pad = (n + 7) // 8 * 8
    act = {"quick_gelu": ops.quick_gelu_, "gelu": ops.gelu_}[hidden_act]
    for i, layer in enumerate(layers):
        (w_qkv, b_qkv), (w_out, b_out), (w_fc1, b_fc1), (w_fc2, b_fc2), ln1, ln2 = weights(prep, layer, i)
        x = ops.layernorm_rows(h, *ln1)
        q = torch.empty((b * n, c), device=dev, dtype=torch.float16)
        k = torch.empty_like(q)
        vt = torch.empty((b, heads, d, n_pad), device=dev, dtype=torch.float16)
        ops.gemm(x, w_qkv, bias=b_qkv, seg_outs=[q, k, vt], seg_width=c, transposed=(0, 0, 1), rows_per_img=n, head_dim=d,
                 tok_pad=n_pad, split_k=split_k)
        a = ops.causal_attention(q, k, vt, b, heads, n) if causal else ops.attention(q, k, vt, b, heads, n, n, d)
        h = ops.gemm(a, w_out, bias=b_out, residual=h, out_f32=f32, split_k=split_k)
        x = ops.layernorm_rows(h, *ln2)
        f = ops.gemm(x, w_fc1, bias=b_fc1, split_k=split_k)
        act(f)
        h = ops.gemm(f, w_fc2, bias=b_fc2, residual=h, out_f32=f32, split_k=split_k)
        if i in keep:
            kept.append(h)
    return (h, kept) if keep else h


class FrozenCLIPEmbedder(nn.Module):
    """Uses the CLIP transformer encoder for text (reference modules.py:88-135), on the sm_90a kernels."""
    LAYERS = [
        "last",
        "pooled",
        "hidden"
    ]

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77, freeze=True, layer="last",
                 layer_idx=None):
        super().__init__()
        assert layer in self.LAYERS
        self.version = version
        self.config = text_config(version)
        self.transformer = _Transformer(self.config)
        self.device = device
        self.max_length = max_length
        if max_length > self.config["max_position_embeddings"]:
            raise ValueError(f"max_length {max_length} exceeds the {self.config['max_position_embeddings']} positions")
        if freeze:
            self.freeze()
        self.layer = layer
        self.layer_idx = layer_idx
        if layer == "hidden":
            assert layer_idx is not None
            assert 0 <= abs(layer_idx) <= 12
        self._tokenizer = None
        self.residual_f32 = True  # the residual-stream precision (False: fp16, for precision studies only)
        self.__dict__["_prep"] = prepare.PrepCache()

    def freeze(self):
        self.transformer = self.transformer.eval()
        for param in self.parameters():
            param.requires_grad = False

    @property
    def tokenizer(self):
        """CLIPTokenizer.from_pretrained(version), built on first use (only the string path needs it)"""
        if self._tokenizer is None:
            try:
                from transformers import CLIPTokenizer
                local = os.path.isdir(str(self.version))  # a local directory is read as it is, never looked up online
                tok = CLIPTokenizer.from_pretrained(self.version, local_files_only=local)
                if tok.vocab_size < 256:  # transformers builds an empty BPE from a directory without vocab.json
                    raise ValueError(f"no byte-level BPE vocabulary found ({tok.vocab_size} tokens)")
                self._tokenizer = tok
            except Exception as e:
                raise RuntimeError(
                    f"FrozenCLIPEmbedder: cannot build the CLIP tokenizer from {self.version!r} ({type(e).__name__}: {e}). "
                    "Pass version=<local directory with vocab.json and merges.txt>, or token ids to encode_tokens()") from e
        return self._tokenizer

    def tokenize(self, text):
        """int64 [B, max_length] token ids on the host (the reference's tokenizer call, modules.py:118-119)"""
        batch_encoding = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                                        return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        return batch_encoding["input_ids"]

    def forward(self, text):
        return self.encode_tokens(self.tokenize(text))

    def encode(self, text):
        return self(text)

    # ---- the encoder on the kernels ------------------------------------------------------------------------------------
    def _depth(self):
        """(number of encoder layers to run, apply final_layer_norm)"""
        n_layers = self.config["num_hidden_layers"]
        if self.layer == "hidden":
            idx = self.layer_idx
            if not -(n_layers + 1) <= idx <= n_layers:
                raise IndexError(f"layer_idx {idx} is out of range for {n_layers + 1} hidden states")
            return idx % (n_layers + 1), False
        return n_layers, True

    def _pooled_rows(self, ids):
        return pooled_rows(ids, self.config["eos_token_id"])

    @torch.no_grad()
    def encode_tokens(self, ids):
        """ids int64 [B, n] (n <= max positions; host or device) -> fp32 [B, n, C] (`pooled`: [B, 1, C]) on the module's
        device, computed on the current stream."""
        tm = self.transformer.text_model
        dev = tm.embeddings.token_embedding.weight.device
        if dev.type != "cuda":
            raise RuntimeError("FrozenCLIPEmbedder runs on the sm_90a kernels only: move the model to a CUDA device")
        if ids.dtype != torch.int64 or ids.dim() != 2:
            raise ValueError(f"token ids must be int64 [B, n], got {ids.dtype} {tuple(ids.shape)}")
        ids_dev = ids.to(dev, non_blocking=False).contiguous()
        b, n = ids_dev.shape
        c, heads = self.config["hidden_size"], self.config["num_attention_heads"]
        depth, final_ln = self._depth()
        f32 = self.residual_f32
        h = ops.clip_embed(ids_dev, tm.embeddings.token_embedding.weight, tm.embeddings.position_embedding.weight, out_f32=f32)
        h = run_layers(tm.encoder.layers[:depth], self._prep, h, b, n, heads, "quick_gelu", causal=True, f32=f32)
        if final_ln:
            ln = tm.final_layer_norm
            h = ops.layernorm_rows(h, ln.weight, ln.bias, ln.eps, out_f32=True)
        elif h.dtype != torch.float32:
            h = h.float()  # fp16 residual stream (precision studies only)
        z = h.view(b, n, c)
        if self.layer == "pooled":
            z = z[torch.arange(b, device=dev), self._pooled_rows(ids_dev)][:, None, :]
        return z
