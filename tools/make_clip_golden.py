"""Generate tests/golden/clip_text_golden.pt with the UNMODIFIED reference's FrozenCLIPEmbedder
(ldm/modules/encoders/modules.py:88-135) running transformers' CLIPTextModel on the CPU in fp32.

    python tools/make_clip_golden.py

tools/ref_shims.install() stands a stub in for the reference's FrozenCLIPEmbedder (the other tools never need CLIP);
this tool loads a second, untouched copy of the reference's modules.py to get the real class, and leaves install() as it
is.  `version` is a temporary directory this tool writes: a CLIPTextConfig plus save_pretrained weights regenerated from
names by oracle/synth.py, and a tokenizer whose vocab.json / merges.txt are synthesized here (every byte, a few merges,
<|startoftext|> and <|endoftext|>).  Nothing is downloaded.

The fixture holds the vocabulary and merges (so tests rebuild the tokenizer without the reference), the prompts, and per
config ("tiny": 2 layers of width 64, one head, the tiny YAMLs' context_dim; "sd15": CLIP ViT-L/14's text tower) the
text config, the token ids and the outputs of layer="last", layer="hidden" with layer_idx=-2 and layer="pooled".  Also
the reference's cond_stage_model.* key list.  Outputs only: the weights are regenerated from names.
"""
import importlib.util
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import save_golden  # noqa: E402
import clip_golden  # noqa: E402

PROMPTS = ["", "a photo of a cat",
           "the photo of the cat on the mat, the cat of the photo, the mat of the cat, a cat and a photo of the "
           "photographer with the camera on the table in the kitchen of the house at the end of the street"]
MERGES = ["t h", "th e</w>", "o f</w>", "c a", "ca t</w>", "p h", "ph o", "pho t", "phot o</w>", "m a", "ma t</w>",
          "a n", "an d</w>", "o n</w>"]


def bytes_to_unicode():
    """the byte -> printable character map of byte-level BPE (GPT-2, CLIP)"""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, map(chr, cs)))


def synth_vocab():
    chars = list(bytes_to_unicode().values())
    toks = chars + [c + "</w>" for c in chars] + [m.replace(" ", "") for m in MERGES] + ["<|startoftext|>", "<|endoftext|>"]
    return {t: i for i, t in enumerate(toks)}


def reference_clip_class():
    """the reference's FrozenCLIPEmbedder from a fresh copy of its module (install() stubs the imported one)"""
    ref_shims.install()
    path = os.path.join(ref_shims.REFERENCE_ROOT, "ldm", "modules", "encoders", "modules.py")
    spec = importlib.util.spec_from_file_location("_reference_encoders_unstubbed", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.FrozenCLIPEmbedder


def text_config(which, vocab):
    eos = vocab["<|endoftext|>"]
    if which == "tiny":
        return {"vocab_size": len(vocab), "hidden_size": 64, "intermediate_size": 256, "num_hidden_layers": 2,
                "num_attention_heads": 1, "max_position_embeddings": 77, "hidden_act": "quick_gelu", "layer_norm_eps": 1e-5,
                "bos_token_id": vocab["<|startoftext|>"], "eos_token_id": eos, "pad_token_id": eos}
    # CLIP ViT-L/14 (openai/clip-vit-large-patch14's text_config, whose eos_token_id is 2: pooled = argmax token id)
    return {"vocab_size": 49408, "hidden_size": 768, "intermediate_size": 3072, "num_hidden_layers": 12,
            "num_attention_heads": 12, "max_position_embeddings": 77, "hidden_act": "quick_gelu", "layer_norm_eps": 1e-5,
            "bos_token_id": 0, "eos_token_id": 2, "pad_token_id": 1}


def run(which, g, Embedder):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = text_config(which, g["vocab"])
    out = {"config": cfg}
    with tempfile.TemporaryDirectory() as d:
        clip_golden.write_version_dir(d, {**g, which: {"config": cfg}}, which)
        model = CLIPTextModel(CLIPTextConfig(**cfg))
        shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(clip_golden.synth_text_weights(shapes), strict=True)
        model.save_pretrained(d)
        del model
        for name, kw in (("last", {}), ("hidden-2", {"layer": "hidden", "layer_idx": -2}), ("pooled", {"layer": "pooled"})):
            emb = Embedder(version=d, device="cpu", **kw)
            with torch.no_grad():
                z = emb.encode(PROMPTS)
            out[name] = z.float().contiguous()
            ids = emb.tokenizer(PROMPTS, truncation=True, max_length=emb.max_length, return_length=True,
                                return_overflowing_tokens=False, padding="max_length", return_tensors="pt")["input_ids"]
            out["ids"] = ids.clone()
            if which == "sd15" and name == "last":
                g["keys"] = ["cond_stage_model." + k for k in emb.state_dict()]
            print(f"{which} {name}: {tuple(z.shape)} |z| {z.norm():.3f}")
    return out


def main():
    torch.manual_seed(0)
    Embedder = reference_clip_class()
    vocab = synth_vocab()
    g = {"vocab": vocab, "merges": list(MERGES), "prompts": list(PROMPTS)}
    g["tiny"] = run("tiny", g, Embedder)
    g["sd15"] = run("sd15", g, Embedder)
    save_golden(g, clip_golden.PATH)
    print(clip_golden.PATH)


if __name__ == "__main__":
    main()
