"""Host-side checks of the MiDaS annotator: the module tree against the reference's state dict, checkpoint loading,
the input domain, and the timm stand-in that tools/make_midas_golden.py runs the reference with, against
transformers' independent DPT-Large implementation."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_io import load_golden  # noqa: E402
import midas_golden as mg  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "midas_golden.pt")


@pytest.fixture(scope="module")
def golden_keys():
    return load_golden(GOLDEN)["keys"]


@pytest.fixture(scope="module")
def model():
    from ctrlora_b200.annotator.midas import DPTDepthModel
    return DPTDepthModel()


def test_state_dict_matches_the_reference(golden_keys, model):
    """MiDaSInference's keys (the fixture records the reference's) are DPTDepthModel's under `model.`, same shapes, same
    order, and the fixture's weights load strictly"""
    ours = [("model." + k, tuple(v.shape)) for k, v in model.state_dict().items()]
    assert ours == [(k, tuple(s)) for k, s in golden_keys]
    assert "model.pretrained.model.head.weight" in dict(ours) and "model.pretrained.model.norm.bias" in dict(ours)
    sd = {k[len("model."):]: v for k, v in mg.weights(dict(golden_keys)).items()}
    model.load_state_dict(sd, strict=True)


def _save(path, sd, wrap):
    torch.save({"model": sd, "optimizer": {"state": {}}} if wrap else sd, path)


@pytest.mark.parametrize("wrap", [False, True])
def test_checkpoint_loading_unwraps_model(tmp_path, golden_keys, wrap):
    """BaseModel.load: a file with an "optimizer" key is read from its "model" entry"""
    from ctrlora_b200.annotator.midas import MiDaSInference
    sd = {k[len("model."):]: torch.full(tuple(s), 0.5) for k, s in golden_keys}
    _save(tmp_path / "dpt_large_384.pt", sd, wrap)
    inf = MiDaSInference("dpt_large", ckpt_dir=str(tmp_path))
    assert torch.equal(inf.model.scratch.layer1_rn.weight, sd["scratch.layer1_rn.weight"])


def test_missing_checkpoint_never_downloads(tmp_path, monkeypatch):
    from ctrlora_b200.annotator.midas import MidasDetector

    def refuse(*a, **k):
        raise AssertionError("network access attempted")
    monkeypatch.setattr(socket.socket, "connect", refuse)
    with pytest.raises(FileNotFoundError, match="dpt_large_384.pt"):
        MidasDetector(ckpt_dir=str(tmp_path), device="cpu")


@pytest.mark.parametrize("model_type", ["dpt_hybrid", "midas_v21", "midas_v21_small"])
def test_other_model_types_are_not_implemented(tmp_path, model_type):
    from ctrlora_b200.annotator.midas import MiDaSInference
    with pytest.raises(NotImplementedError):
        MiDaSInference(model_type, ckpt_dir=str(tmp_path))


def test_other_configurations_are_not_implemented():
    from ctrlora_b200.annotator.midas import DPTDepthModel
    with pytest.raises(NotImplementedError):
        DPTDepthModel(backbone="vitb_rn50_384")
    with pytest.raises(NotImplementedError):
        DPTDepthModel(non_negative=False)


@pytest.mark.parametrize("h,w,ok", [(384, 384, True), (200, 328, True), (32, 32, True), (31, 64, False),
                                    (48, 64, False), (64, 80, False), (16, 64, False)])
def test_domain_and_output_size(model, h, w, ok):
    """gh = H // 16 and gw = W // 16 must be even and >= 2; the depth is 16 gh x 16 gw.  Out-of-domain input raises
    ValueError before anything reaches a device (the model here is on the CPU)"""
    x = torch.zeros(1, 3, h, w)
    if ok:
        gh, gw = model.grid(x)
        assert (16 * gh, 16 * gw) == (h // 16 * 16, w // 16 * 16)
        with pytest.raises(RuntimeError, match="CUDA"):
            model(x)
    else:
        with pytest.raises(ValueError):
            model(x)


def test_fixture_is_not_vacuous():
    """the synthetic weights give a positive, varied depth and a normal map with structure"""
    g = load_golden(GOLDEN)
    for size in mg.SIZES:
        d = mg.unband(g[f"{size}.depth"])
        assert (d > 0).float().mean() > 0.9 and d.std() > 0.1 * d.mean()
        n8 = mg.unband(g[f"{size}.normal_u8"]).numpy()
        assert len(np.unique(n8[..., 0])) > 100 and len(np.unique(mg.unband(g[f"{size}.depth_u8"]).numpy())) > 100


def _hf_state_dict(ref):
    """the reference DPTDepthModel's weights under transformers' DPTForDepthEstimation names"""
    sd = ref.state_dict()
    out = {}
    vit = "pretrained.model."
    out["dpt.embeddings.cls_token"] = sd[vit + "cls_token"]
    out["dpt.embeddings.position_embeddings"] = sd[vit + "pos_embed"]
    out["dpt.embeddings.patch_embeddings.projection.weight"] = sd[vit + "patch_embed.proj.weight"]
    out["dpt.embeddings.patch_embeddings.projection.bias"] = sd[vit + "patch_embed.proj.bias"]
    out["dpt.layernorm.weight"], out["dpt.layernorm.bias"] = sd[vit + "norm.weight"], sd[vit + "norm.bias"]
    for i in range(24):
        p, q = f"{vit}blocks.{i}.", f"dpt.encoder.layer.{i}."
        qw, qb = sd[p + "attn.qkv.weight"].chunk(3), sd[p + "attn.qkv.bias"].chunk(3)
        for j, n in enumerate(("query", "key", "value")):
            out[q + f"attention.attention.{n}.weight"], out[q + f"attention.attention.{n}.bias"] = qw[j], qb[j]
        for src, dst in (("attn.proj", "attention.output.dense"), ("norm1", "layernorm_before"),
                         ("norm2", "layernorm_after"), ("mlp.fc1", "intermediate.dense"), ("mlp.fc2", "output.dense")):
            out[q + dst + ".weight"], out[q + dst + ".bias"] = sd[p + src + ".weight"], sd[p + src + ".bias"]
    for k in range(4):
        pp = f"pretrained.act_postprocess{k + 1}."
        out[f"neck.reassemble_stage.readout_projects.{k}.0.weight"] = sd[pp + "0.project.0.weight"]
        out[f"neck.reassemble_stage.readout_projects.{k}.0.bias"] = sd[pp + "0.project.0.bias"]
        out[f"neck.reassemble_stage.layers.{k}.projection.weight"] = sd[pp + "3.weight"]
        out[f"neck.reassemble_stage.layers.{k}.projection.bias"] = sd[pp + "3.bias"]
        if k != 2:
            out[f"neck.reassemble_stage.layers.{k}.resize.weight"] = sd[pp + "4.weight"]
            out[f"neck.reassemble_stage.layers.{k}.resize.bias"] = sd[pp + "4.bias"]
        out[f"neck.convs.{k}.weight"] = sd[f"scratch.layer{k + 1}_rn.weight"]
        # transformers' fusion layers run from the deepest: fusion_stage.layers.0 is refinenet4
        rf, fl = f"scratch.refinenet{4 - k}.", f"neck.fusion_stage.layers.{k}."
        out[fl + "projection.weight"], out[fl + "projection.bias"] = sd[rf + "out_conv.weight"], sd[rf + "out_conv.bias"]
        for r in (1, 2):
            for c in (1, 2):
                for t in ("weight", "bias"):
                    out[fl + f"residual_layer{r}.convolution{c}.{t}"] = sd[rf + f"resConfUnit{r}.conv{c}.{t}"]
    for src, dst in (("0", "head.head.0"), ("2", "head.head.2"), ("4", "head.head.4")):
        for t in ("weight", "bias"):
            out[f"{dst}.{t}"] = sd[f"scratch.output_conv.{src}.{t}"]
    return out


def test_timm_stand_in_against_transformers_dpt():
    """the reference DPTDepthModel built on tools/ref_shims.py's timm stand-in computes what transformers'
    DPTForDepthEstimation (an independent DPT-Large implementation) computes with the same weights: this is what makes
    the fixture trustworthy"""
    transformers = pytest.importorskip("transformers")
    from tools import ref_shims
    if not os.path.isdir(os.path.join(ref_shims.REFERENCE_ROOT, "annotator", "midas")):
        pytest.skip("the reference tree is not present")
    ref_shims.install_timm_shim()
    if ref_shims.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.midas.midas.dpt_depth import DPTDepthModel
    torch.manual_seed(0)
    ref = DPTDepthModel(path=None, backbone="vitl16_384", non_negative=True).eval()
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    ref.load_state_dict({k[len("model."):]: v for k, v in mg.weights({"model." + k: s for k, s in shapes.items()}).items()})
    cfg = transformers.DPTConfig(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096,
                                 image_size=384, patch_size=16, layer_norm_eps=1e-6, backbone_out_indices=[5, 11, 17, 23],
                                 neck_hidden_sizes=[256, 512, 1024, 1024], fusion_hidden_size=256, readout_type="project",
                                 reassemble_factors=[4, 2, 1, 0.5], is_hybrid=False, head_in_index=-1,
                                 use_batch_norm_in_fusion_residual=False, add_projection=False)
    hf = transformers.DPTForDepthEstimation(cfg).eval()
    missing, unexpected = hf.load_state_dict(_hf_state_dict(ref), strict=False)
    assert not unexpected and not [k for k in missing if "running" not in k], (missing, unexpected)
    x = mg.image_tensor(mg.image((64, 64)))  # square: transformers reshapes a non-hybrid grid as size x size
    with torch.no_grad():
        a = ref(x)
        b = hf(pixel_values=x).predicted_depth
    assert a.shape == b.shape == (1, 64, 64)
    err = ((a - b).norm() / a.norm()).item()
    assert err < 1e-5, err


def test_launch_references_against_restatements():
    """tests/midas_launches.py's references at tiny shapes against independent restatements: index loops for the patch
    gather and the depth-to-space, F.conv_transpose2d for a kernel = stride transposed conv as depth-to-space of a
    matrix product"""
    import midas_launches as ML
    g = torch.Generator().manual_seed(5)
    px = torch.randn(2, 3, 35, 50, generator=g)
    got = ML.patch_gather_hw(px, 16, 776).float()
    for b in range(2):
        for py in range(2):
            for qx in range(3):
                row = got[b * 6 + py * 3 + qx]
                want = px[b, :, 16 * py:16 * py + 16, 16 * qx:16 * qx + 16].reshape(-1).half().float()
                assert torch.equal(row[:768], want) and not row[768:].any()
    x = torch.randn(1, 3, 5, 8, generator=g)
    wt = torch.randn(8, 8, 2, 2, generator=g)
    bias = torch.randn(8, generator=g)
    src = (x.reshape(-1, 8) @ wt.permute(2, 3, 1, 0).reshape(32, 8).t()).view(1, 3, 5, 32)
    d2s = ML.depth_to_space_bias(src, bias, 2).float()
    ref = F_conv_t(x, wt, bias)
    assert (d2s - ref).abs().max().item() <= 2 ** -10 * ref.abs().max().item()
    for y in range(6):
        for xx in range(10):
            ky, kx = y % 2, xx % 2
            want = (src[0, y // 2, xx // 2, (ky * 2 + kx) * 8:(ky * 2 + kx + 1) * 8] + bias).half()
            assert torch.equal(d2s[0, y, xx].half(), want)


def F_conv_t(x, wt, bias):
    """ConvTranspose2d(kernel = stride = 2) of NHWC x -> NHWC"""
    import torch.nn.functional as F
    return F.conv_transpose2d(x.permute(0, 3, 1, 2), wt, bias, stride=2).permute(0, 2, 3, 1)
