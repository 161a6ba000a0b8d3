"""The CLIP text-encoder fixture (tests/golden/clip_text_golden.pt, written by tools/make_clip_golden.py from the
unmodified reference's FrozenCLIPEmbedder) and what the tests rebuild from it: a `version` directory with the
fixture's tokenizer vocabulary and text config, and the name-keyed synthetic weights (oracle/synth.py)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from golden_io import load_golden  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "clip_text_golden.pt")
SEED = 0
WEIGHT_PREFIX = "cond_stage_model.transformer."  # synth RNG key of a weight: this + its CLIPTextModel name


def load():
    return load_golden(PATH)


def write_version_dir(path, g, which):
    """A `version` directory for FrozenCLIPEmbedder / CLIPTokenizer: vocab.json, merges.txt and config.json of the
    fixture's `which` ("tiny" or "sd15") config.  Returns path."""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "vocab.json"), "w") as f:
        json.dump(g["vocab"], f)
    with open(os.path.join(path, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n" + "\n".join(g["merges"]) + "\n")
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(g[which]["config"], f)
    return path


def synth_text_weights(shapes, seed=SEED):
    """{CLIPTextModel key (text_model.*): fp32 tensor} regenerated from names"""
    return {k: synth.synth_param(WEIGHT_PREFIX + k, s, seed) for k, s in shapes.items()}


def embedder_weights(embedder, seed=SEED):
    """the synthetic weights as a state dict of a FrozenCLIPEmbedder (keys transformer.text_model.*)"""
    shapes = {k[len("transformer."):]: tuple(v.shape) for k, v in embedder.state_dict().items()}
    return {"transformer." + k: v for k, v in synth_text_weights(shapes, seed).items()}
