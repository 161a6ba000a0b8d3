"""The image-prompt models' host side without a GPU: state-dict keys and shapes against transformers' and the reference
app's (tests/golden/clip_vision_golden.pt), the position_ids buffer of older checkpoints, config parsing and the
configs the kernels refuse, from_pretrained from a local directory (safetensors, .bin, a full CLIPModel checkpoint), and
that none of it touches the network."""
import json
import os
import socket

import pytest
import torch

import clip_vision_golden as cvg


@pytest.fixture(scope="module")
def g():
    return cvg.load()


def _meta(cls, *a, **kw):
    with torch.device("meta"):
        return cls(*a, **kw)


def _shapes(model):
    return [(k, tuple(v.shape)) for k, v in model.state_dict().items()]


def test_vision_keys_and_shapes(g):
    from ctrlora_b200.image_encoder import CLIPVisionModelWithProjection
    model = _meta(CLIPVisionModelWithProjection)  # the built-in default: the IP-Adapter SD1.5 image encoder
    assert list(model.state_dict()) == g["vision_sd15"]["keys"]
    sd = model.state_dict()
    assert sd["vision_model.embeddings.patch_embedding.weight"].shape == (1280, 3, 14, 14)
    assert sd["vision_model.embeddings.position_embedding.weight"].shape == (257, 1280)
    assert sd["vision_model.encoder.layers.31.mlp.fc1.weight"].shape == (5120, 1280)
    assert sd["visual_projection.weight"].shape == (1024, 1280)
    tiny = _meta(CLIPVisionModelWithProjection, g["vision_tiny"]["config"])
    assert list(tiny.state_dict()) == g["vision_tiny"]["keys"]
    assert tiny.state_dict()["visual_projection.weight"].shape == (64, 160)
    assert all(not p.requires_grad for p in model.parameters()) and not model.training


def test_text_and_projection_keys(g):
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection, ImageProjModel
    text = _meta(CLIPTextModelWithProjection)  # built-in: the ViT-H/14 text tower
    assert list(text.state_dict()) == g["text_sd15"]["keys"]
    assert text.state_dict()["text_projection.weight"].shape == (1024, 1024)
    assert text.config["hidden_act"] == "gelu" and text.config["num_hidden_layers"] == 24
    tiny = _meta(CLIPTextModelWithProjection, g["text_tiny"]["config"])
    assert list(tiny.state_dict()) == g["text_tiny"]["keys"]
    proj = ImageProjModel()
    assert list(proj.state_dict()) == g["vision_sd15"]["proj_keys"]
    assert proj.proj.weight.shape == (3072, 1024) and proj.norm.weight.shape == (768,)
    # the ip-adapter_sd15.bin "image_proj" entry loads strictly
    proj.load_state_dict(cvg.weights(proj, "proj"), strict=True)


def test_position_ids_accepted():
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection, CLIPVisionModelWithProjection
    cfg = dict(cvg.VISION["tiny"], num_hidden_layers=1)
    model = CLIPVisionModelWithProjection(cfg)
    sd = cvg.weights(model, "vision")
    sd["vision_model.embeddings.position_ids"] = torch.arange(257)[None]
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.vision_model.embeddings.class_embedding, sd["vision_model.embeddings.class_embedding"])
    text = CLIPTextModelWithProjection({"vocab_size": 300, "hidden_size": 64, "intermediate_size": 128,
                                        "num_hidden_layers": 1, "num_attention_heads": 1, "projection_dim": 32})
    sd = cvg.weights(text, "text")
    sd["text_model.embeddings.position_ids"] = torch.arange(77)[None]
    text.load_state_dict(sd, strict=True)


def test_config_parsing():
    from ctrlora_b200 import image_encoder as ie
    assert ie.vision_config() == ie.VIT_H_VISION_CONFIG
    # a CLIPConfig: the tower's own entry is used
    clip = {"projection_dim": 512, "vision_config": {"hidden_size": 160, "num_attention_heads": 2, "projection_dim": 64},
            "text_config": {"hidden_size": 128, "num_attention_heads": 2, "hidden_act": "quick_gelu"}}
    v = ie.vision_config(clip)
    assert v["hidden_size"] == 160 and v["projection_dim"] == 64 and v["num_hidden_layers"] == 32
    t = ie.text_config(clip)
    assert t["hidden_size"] == 128 and t["hidden_act"] == "quick_gelu" and t["projection_dim"] == 1024
    from transformers import CLIPVisionConfig
    assert ie.vision_config(CLIPVisionConfig(**cvg.VISION["tiny"])) == cvg.VISION["tiny"]


@pytest.mark.parametrize("bad,match", [
    ({"hidden_act": "relu"}, "hidden_act"),
    ({"hidden_act": "gelu_new"}, "hidden_act"),
    ({"hidden_size": 1200, "num_attention_heads": 16}, "head size"),   # 75, not a multiple of 8
    ({"hidden_size": 2048, "num_attention_heads": 8}, "head size"),    # 256 > 160
    ({"image_size": 225}, "patch size"),
])
def test_vision_config_refused(bad, match):
    from ctrlora_b200.image_encoder import CLIPVisionModelWithProjection
    with pytest.raises(ValueError, match=match):
        _meta(CLIPVisionModelWithProjection, bad)


@pytest.mark.parametrize("bad,match", [({"hidden_act": "relu"}, "hidden_act"), ({"num_attention_heads": 8}, "head size"),
                                       ({"max_position_embeddings": 256}, "positions")])
def test_text_config_refused(bad, match):
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection
    with pytest.raises(ValueError, match=match):
        _meta(CLIPTextModelWithProjection, bad)


def test_outputs_refused_without_a_gpu():
    from ctrlora_b200.image_encoder import CLIPVisionModelWithProjection, ImageProjModel
    model = CLIPVisionModelWithProjection(dict(cvg.VISION["tiny"], num_hidden_layers=1))
    with pytest.raises(NotImplementedError, match="output_hidden_states"):
        model(cvg.pixels(1), output_hidden_states=True)
    with pytest.raises(RuntimeError, match="CUDA device"):
        model(cvg.pixels(1))
    with pytest.raises(RuntimeError, match="CUDA device"):
        ImageProjModel(64, 64)(torch.zeros(1, 64))


@pytest.mark.parametrize("fmt", ["safetensors", "bin", "clip_bin"])
def test_from_pretrained_local(tmp_path, fmt):
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection, CLIPVisionModelWithProjection
    vcfg = dict(cvg.VISION["tiny"], num_hidden_layers=1)
    tcfg = {"vocab_size": 300, "hidden_size": 64, "intermediate_size": 128, "num_hidden_layers": 1,
            "num_attention_heads": 1, "projection_dim": 32, "hidden_act": "gelu"}
    vis, txt = CLIPVisionModelWithProjection(vcfg), CLIPTextModelWithProjection(tcfg)
    vsd, tsd = cvg.weights(vis, "vision"), cvg.weights(txt, "text")
    d = str(tmp_path)
    if fmt == "clip_bin":  # a full CLIPModel checkpoint (both towers, logit_scale) and a CLIPConfig
        cfg = {"model_type": "clip", "projection_dim": 32, "vision_config": vcfg, "text_config": tcfg}
        torch.save({**vsd, **tsd, "logit_scale": torch.tensor(2.6592)}, os.path.join(d, "pytorch_model.bin"))
    else:
        cfg = vcfg
        if fmt == "safetensors":
            from safetensors.torch import save_file
            save_file(vsd, os.path.join(d, "model.safetensors"))
        else:
            torch.save(vsd, os.path.join(d, "pytorch_model.bin"))
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(cfg, f)
    loaded = CLIPVisionModelWithProjection.from_pretrained(d)
    assert loaded.config["hidden_size"] == 160
    for k, v in loaded.state_dict().items():
        assert torch.equal(v, vsd[k]), k
    if fmt == "clip_bin":
        t = CLIPTextModelWithProjection.from_pretrained(d)
        assert t.config["hidden_size"] == 64
        assert torch.equal(t.text_projection.weight, tsd["text_projection.weight"])


def test_from_pretrained_refuses_a_hub_name(tmp_path):
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection, CLIPVisionModelWithProjection
    with pytest.raises(OSError, match="not a local directory"):
        CLIPVisionModelWithProjection.from_pretrained("h94/IP-Adapter")
    with pytest.raises(OSError, match="not a local directory"):
        CLIPTextModelWithProjection.from_pretrained("laion/CLIP-ViT-H-14-laion2B-s32B-b79K")
    with pytest.raises(OSError, match="config.json"):
        CLIPVisionModelWithProjection.from_pretrained(str(tmp_path))


def test_attention_mask_must_be_right_padding():
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection
    text = CLIPTextModelWithProjection({"vocab_size": 300, "hidden_size": 64, "intermediate_size": 128,
                                        "num_hidden_layers": 1, "num_attention_heads": 1, "projection_dim": 32})
    ids = torch.ones((2, 5), dtype=torch.int64)
    for mask in ([[1, 1, 0, 1, 0], [1, 1, 1, 1, 1]], [[0, 1, 1, 1, 1], [1, 1, 1, 1, 1]], [[1, 1, 2, 0, 0], [1] * 5]):
        with pytest.raises(ValueError, match="right padding"):
            text(ids, attention_mask=torch.tensor(mask))


def test_building_touches_no_network(monkeypatch, tmp_path):
    calls = []

    def refuse(*a, **k):
        calls.append(a)
        raise OSError("network access attempted")

    monkeypatch.setattr(socket.socket, "connect", refuse)
    monkeypatch.setattr(socket, "create_connection", refuse)
    monkeypatch.setattr(socket, "getaddrinfo", refuse)
    from ctrlora_b200.image_encoder import CLIPTextModelWithProjection, CLIPVisionModelWithProjection, ImageProjModel
    model = CLIPVisionModelWithProjection(dict(cvg.VISION["tiny"], num_hidden_layers=1))
    d = str(tmp_path)
    torch.save(cvg.weights(model, "vision"), os.path.join(d, "pytorch_model.bin"))
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(model.config, f)
    CLIPVisionModelWithProjection.from_pretrained(d)
    _meta(CLIPVisionModelWithProjection)
    _meta(CLIPTextModelWithProjection)
    ImageProjModel()
    with pytest.raises(OSError):
        CLIPVisionModelWithProjection.from_pretrained("h94/IP-Adapter")
    assert not calls
