"""The CLIP text encoder's host side without a GPU: state-dict keys against the reference's, the tokenizer rebuilt from
the fixture's vocabulary, the per-model opt-in of create_model (a default model keeps cond_stage_model None), checkpoint
key handling, and that building an encoder touches no network."""
import glob
import os
import socket

import pytest
import torch

import clip_golden

ROOT = clip_golden.ROOT
CONFIGS = sorted(glob.glob(os.path.join(ROOT, "configs", "*.yaml")) + glob.glob(os.path.join(ROOT, "tests", "golden", "*.yaml")))
TINY = os.path.join(ROOT, "tests", "golden", "tiny_finetune.yaml")


@pytest.fixture(scope="module")
def g():
    return clip_golden.load()


def _create(path, **kw):
    from ctrlora_b200 import dropin
    dropin.activate()
    from cldm.model import create_model
    return create_model(path, init_weights=False, **kw)


def test_keys_match_the_reference(g):
    model = _create(TINY, text_encoder=True)  # the built-in CLIP ViT-L/14 architecture, nothing fetched
    keys = [k for k in model.state_dict() if k.startswith("cond_stage_model.")]
    assert keys == g["keys"]
    sd = model.cond_stage_model.state_dict()
    assert sd["transformer.text_model.embeddings.token_embedding.weight"].shape == (49408, 768)
    assert sd["transformer.text_model.encoder.layers.11.mlp.fc1.weight"].shape == (3072, 768)
    assert all(not p.requires_grad for p in model.cond_stage_model.parameters())
    assert not model.cond_stage_model.training


def test_position_ids_in_a_checkpoint_are_accepted(g):
    from ctrlora_b200.text_encoder import FrozenCLIPEmbedder
    from ctrlora_b200 import checkpoint
    enc = FrozenCLIPEmbedder()
    sd = clip_golden.embedder_weights(enc)
    sd["transformer.text_model.embeddings.position_ids"] = torch.arange(77)[None]
    enc.load_state_dict(sd, strict=True)
    w = enc.transformer.text_model.encoder.layers[3].self_attn.q_proj.weight
    assert torch.equal(w, sd["transformer.text_model.encoder.layers.3.self_attn.q_proj.weight"])
    # checkpoint_weights: an opted-in model keeps its CLIP keys and drops position_ids; any other model drops them all
    expected = {"a.w": torch.zeros(2), **{"cond_stage_model." + k: v for k, v in enc.state_dict().items()}}
    file = {"a.w": torch.ones(2), **{"cond_stage_model." + k: v for k, v in sd.items()}}
    kept = checkpoint.checkpoint_weights(file, expected)
    assert set(kept) == set(expected)
    assert set(checkpoint.checkpoint_weights(file, {"a.w": torch.zeros(2)})) == {"a.w"}
    del file["cond_stage_model.transformer.text_model.final_layer_norm.bias"]
    with pytest.raises(ValueError, match="missing"):
        checkpoint.checkpoint_weights(file, expected)


@pytest.mark.parametrize("which", ["tiny", "sd15"])
def test_tokenizer_from_fixture_vocabulary(g, which, tmp_path):
    from ctrlora_b200.text_encoder import FrozenCLIPEmbedder
    d = clip_golden.write_version_dir(str(tmp_path / which), g, which)
    enc = FrozenCLIPEmbedder(version=d)
    ids = enc.tokenize(g["prompts"])
    assert ids.dtype == torch.int64 and ids.shape == (3, 77)
    assert torch.equal(ids, g[which]["ids"])
    eos = g["vocab"]["<|endoftext|>"]
    assert ids[0, 1] == eos and ids[2, -1] == eos and (ids[2, 1:-1] != eos).all()  # the long prompt is truncated at 77
    assert enc.config["hidden_size"] == g[which]["config"]["hidden_size"]


def test_tokenizer_failure_is_clear(tmp_path):
    from ctrlora_b200.text_encoder import FrozenCLIPEmbedder
    enc = FrozenCLIPEmbedder(version=str(tmp_path))  # an empty local directory: built-in config, no tokenizer files
    with pytest.raises(RuntimeError, match="CLIP tokenizer"):
        enc.tokenize(["a cat"])


def test_opt_in_is_per_model(g, tmp_path):
    d = clip_golden.write_version_dir(str(tmp_path / "tiny"), g, "tiny")
    opted = _create(TINY, text_encoder={"version": d, "layer": "hidden", "layer_idx": -2})
    enc = opted.cond_stage_model
    assert type(enc).__name__ == "FrozenCLIPEmbedder" and enc.layer == "hidden" and enc.layer_idx == -2
    assert enc.config["hidden_size"] == 64
    for path in CONFIGS:
        model = _create(path)
        assert model.cond_stage_model is None, path
        assert not any(k.startswith("cond_stage_model.") for k in model.state_dict()), path
        del model
    from ctrlora_b200 import checkpoint
    assert checkpoint.IGNORED_PREFIXES == ("cond_stage_model.",)


def test_building_touches_no_network(monkeypatch):
    calls = []

    def refuse(*a, **k):
        calls.append(a)
        raise OSError("network access attempted")

    monkeypatch.setattr(socket.socket, "connect", refuse)
    monkeypatch.setattr(socket, "create_connection", refuse)
    monkeypatch.setattr(socket, "getaddrinfo", refuse)
    model = _create(TINY, text_encoder=True)
    assert model.cond_stage_model is not None
    assert model.cond_stage_model._tokenizer is None  # built lazily, on the first call with strings
    assert not calls
