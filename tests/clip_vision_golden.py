"""The IP-Adapter image-encoder fixture (tests/golden/clip_vision_golden.pt, written by tools/make_clip_vision_golden.py
from transformers' CLIPVisionModelWithProjection / CLIPTextModelWithProjection and the reference app's ImageProjModel, fp32
on the CPU) and what the tests rebuild from it: the configs, the name-keyed synthetic weights and pixels
(oracle/synth.py), and a tokenizer directory from the CLIP text fixture's vocabulary."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from golden_io import load_golden  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "clip_vision_golden.pt")
SEED = 0
BATCH = 2
# synth RNG key of a weight: prefix + its transformers / ImageProjModel name
PREFIX = {"vision": "image_encoder.", "text": "text_encoder.", "proj": "image_proj."}

VISION = {
    # d_head 80 and 257 tokens like ViT-H/14, 2 layers; projection 64 = tests/golden/tiny_style.yaml's context_dim
    "tiny": {"hidden_size": 160, "intermediate_size": 640, "num_hidden_layers": 2, "num_attention_heads": 2,
             "num_channels": 3, "image_size": 224, "patch_size": 14, "projection_dim": 64, "hidden_act": "gelu",
             "layer_norm_eps": 1e-5},
    # the IP-Adapter SD1.5 image_encoder, CLIP ViT-H/14
    "sd15": {"hidden_size": 1280, "intermediate_size": 5120, "num_hidden_layers": 32, "num_attention_heads": 16,
             "num_channels": 3, "image_size": 224, "patch_size": 14, "projection_dim": 1024, "hidden_act": "gelu",
             "layer_norm_eps": 1e-5},
}
PROJ = {"tiny": {"cross_attention_dim": 64, "clip_embeddings_dim": 64, "clip_extra_context_tokens": 4},
        "sd15": {"cross_attention_dim": 768, "clip_embeddings_dim": 1024, "clip_extra_context_tokens": 4}}


def text_config(which, vocab):
    if which == "tiny":
        eos = vocab["<|endoftext|>"]
        return {"vocab_size": len(vocab), "hidden_size": 64, "intermediate_size": 256, "num_hidden_layers": 2,
                "num_attention_heads": 1, "max_position_embeddings": 77, "hidden_act": "gelu", "layer_norm_eps": 1e-5,
                "projection_dim": 64, "bos_token_id": vocab["<|startoftext|>"], "eos_token_id": eos, "pad_token_id": eos}
    # the ViT-H/14 text tower (laion2B), eos_token_id 2: the pooled row is the argmax token id
    return {"vocab_size": 49408, "hidden_size": 1024, "intermediate_size": 4096, "num_hidden_layers": 24,
            "num_attention_heads": 16, "max_position_embeddings": 77, "hidden_act": "gelu", "layer_norm_eps": 1e-5,
            "projection_dim": 1024, "bos_token_id": 0, "eos_token_id": 2, "pad_token_id": 1}


def load():
    return load_golden(PATH)


def pixels(batch, seed=SEED, size=224):
    """normalized pixel values fp32 [batch, 3, size, size] (CLIPImageProcessor's output scale)"""
    return synth.synth_input("clip_pixels", (batch, 3, size, size), seed)


def weights(model, kind, seed=SEED):
    """synthetic weights for every key of `model`'s state dict; kind: "vision", "text" or "proj" """
    return {k: synth.synth_param(PREFIX[kind] + k, tuple(v.shape), seed) for k, v in model.state_dict().items()}


def tokenizer_dir(path, vocab, merges):
    """vocab.json and merges.txt for transformers' CLIPTokenizer; returns path"""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "vocab.json"), "w") as f:
        json.dump(vocab, f)
    with open(os.path.join(path, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n" + "\n".join(merges) + "\n")
    return path


def tokenize(path, prompts):
    """the fixture's token ids and attention mask: right padding to the longest prompt, truncation at 77"""
    from transformers import CLIPTokenizer
    tok = CLIPTokenizer.from_pretrained(path, local_files_only=True)
    enc = tok(prompts, padding=True, truncation=True, max_length=77, return_tensors="pt")
    return enc["input_ids"], enc["attention_mask"]
