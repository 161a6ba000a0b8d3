"""Generate tests/golden/clip_vision_golden.pt: what the reference's style app computes for its image prompt
(app/gradio_ctrlora_style_transfer.py:385-409), in fp32 on the CPU.

    python tools/make_clip_vision_golden.py

- transformers' CLIPVisionModelWithProjection gives image_embeds (and, for the tiny config, last_hidden_state);
- the reference's ImageProjModel, taken from an unmodified copy of the app file at run time (only that class's AST node
  is compiled: the rest of the app needs gradio and checkpoints), gives the cond tokens and the uncond tokens of
  torch.zeros_like(image_embeds);
- transformers' CLIPTextModelWithProjection gives text_embeds for the CLIP text fixture's prompts, right-padded with
  an attention mask, as the negative content prompt does.

Configs and the batch are in tests/clip_vision_golden.py: "tiny" (width 160, 2 heads so d_head 80, 257 tokens, 2 layers,
projection 64) and "sd15" (the IP-Adapter's ViT-H/14 image encoder, 32 layers, batch 2); text towers "tiny" (width 64) and
"sd15" (ViT-H/14's 24-layer text tower).  Weights and pixels are regenerated from names by oracle/synth.py; the fixture
holds outputs, token ids, key lists and the transformers version only.  Running it twice writes identical bytes.
"""
import ast
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
import clip_vision_golden as cvg  # noqa: E402


def reference_image_proj_class():
    """ImageProjModel from the unmodified app file: its ClassDef node compiled on its own"""
    path = os.path.join(ref_shims.REFERENCE_ROOT, "app", "gradio_ctrlora_style_transfer.py")
    with open(path) as f:
        tree = ast.parse(f.read(), filename=path)
    node = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "ImageProjModel")
    ns = {"torch": torch}
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return ns["ImageProjModel"]


def run_vision(which, ImageProjModel):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    model = CLIPVisionModelWithProjection(CLIPVisionConfig(**cvg.VISION[which])).eval()
    model.load_state_dict(cvg.weights(model, "vision"), strict=True)
    proj = ImageProjModel(**cvg.PROJ[which]).eval()
    proj.load_state_dict(cvg.weights(proj, "proj"), strict=True)
    with torch.no_grad():
        out = model(cvg.pixels(cvg.BATCH))
        emb = out.image_embeds
        res = {"config": dict(cvg.VISION[which]), "image_embeds": emb.contiguous(), "tokens": proj(emb).contiguous(),
               "uncond_tokens": proj(torch.zeros_like(emb)).contiguous(), "keys": list(model.state_dict()),
               "proj_keys": list(proj.state_dict())}
        if which == "tiny":
            res["last_hidden_state"] = out.last_hidden_state.contiguous()
    print(f"vision {which}: image_embeds {tuple(emb.shape)} |e| {emb.norm():.3f}, tokens |t| {res['tokens'].norm():.3f}")
    return res


def run_text(which, g, tok_dir):
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    cfg = cvg.text_config(which, g["vocab"])
    model = CLIPTextModelWithProjection(CLIPTextConfig(**cfg)).eval()
    model.load_state_dict(cvg.weights(model, "text"), strict=True)
    ids, mask = cvg.tokenize(tok_dir, g["prompts"])
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=mask)
    res = {"config": cfg, "ids": ids.clone(), "attention_mask": mask.clone(), "text_embeds": out.text_embeds.contiguous(),
           "keys": list(model.state_dict())}
    print(f"text {which}: ids {tuple(ids.shape)}, text_embeds |e| {out.text_embeds.norm():.3f}")
    return res


def main():
    import transformers
    torch.manual_seed(0)
    torch.use_deterministic_algorithms(True)
    ImageProjModel = reference_image_proj_class()
    text_fixture = clip_golden.load()
    g = {"transformers_version": transformers.__version__, "batch": cvg.BATCH, "prompts": list(text_fixture["prompts"])}
    for which in ("tiny", "sd15"):
        g["vision_" + which] = run_vision(which, ImageProjModel)
    with tempfile.TemporaryDirectory() as d:
        cvg.tokenizer_dir(d, text_fixture["vocab"], text_fixture["merges"])
        for which in ("tiny", "sd15"):
            g["text_" + which] = run_text(which, text_fixture, d)
    save_golden(g, cvg.PATH)
    print(cvg.PATH)


if __name__ == "__main__":
    main()
