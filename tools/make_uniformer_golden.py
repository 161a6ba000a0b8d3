"""Generate tests/golden/uniformer_golden.pt: what the reference's UniFormer segmentation annotator computes, in fp32
on the CPU.

    python tools/make_uniformer_golden.py

The unmodified reference `annotator.uniformer` (its vendored mmcv and mmseg) is imported from the reference tree with
tools/ref_shims.py's stand-ins for addict, yapf, prettytable, timm.models.layers and matplotlib.  The segmentor is
built by `init_segmentor(exp/upernet_global_small/config.py, None, device="cpu")` and loaded (strict) with
tests/uniformer_golden.py's synthetic weights; `inference_segmentor` and `show_result_pyplot(..., get_palette('ade'),
opacity=1)` then run as written, which is UniformerDetector.__call__ without the checkpoint download.  Per size the
fixture stores the network input size, the four backbone features and the 1/4-level logits at sampled positions, and in
row bands the labels, the RGB map and the top-two margin of the fp32 logits at the input size (the logits resized
twice as the reference resizes them, recomputed here from the captured 1/4-level logits; their argmax is checked
against the reference's labels).  Also the state-dict keys and shapes and get_palette('ade'), as data.  Running it twice
writes identical bytes.
"""
import os
import sys

import cv2
import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import save_golden  # noqa: E402
import uniformer_golden as ug  # noqa: E402


def reference_segmentor():
    """(segmentor on the CPU with the fixture's weights, inference_segmentor, show_result_pyplot, get_palette)"""
    ref_shims.install_uniformer_shims()
    if ref_shims.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.uniformer.mmseg.apis import inference_segmentor, init_segmentor, show_result_pyplot
    from annotator.uniformer.mmseg.core.evaluation import get_palette
    from annotator.uniformer.mmseg.datasets import ADE20KDataset
    cfg = os.path.join(ref_shims.REFERENCE_ROOT, "annotator", "uniformer", "exp", "upernet_global_small", "config.py")
    model = init_segmentor(cfg, None, device="cpu")
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    bn_names = [n for n, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    model.load_state_dict(ug.weights(shapes, bn_names), strict=True)
    model.CLASSES, model.PALETTE = ADE20KDataset.CLASSES, get_palette("ade")
    return model.eval(), inference_segmentor, show_result_pyplot, get_palette


def run(model, infer, show, palette, size):
    img = ug.image(size)
    got = {}
    hooks = [model.backbone.register_forward_pre_hook(lambda m, i: got.__setitem__("input", i[0].detach().clone())),
             model.backbone.register_forward_hook(lambda m, i, o: got.__setitem__("features", [t.detach().clone() for t in o])),
             model.decode_head.conv_seg.register_forward_hook(lambda m, i, o: got.__setitem__("logits", o.detach().clone()))]
    result = infer(model, img)
    rgb = show(model, img, result, palette, opacity=1)
    for h in hooks:
        h.remove()
    labels = torch.from_numpy(result[0].astype(np.int64))
    net = tuple(got["input"].shape[2:])
    # the reference's two logit resizes (EncoderDecoder.encode_decode, then whole_inference's rescale), fp32
    up = F.interpolate(got["logits"], size=net, mode="bilinear", align_corners=False)
    up = F.interpolate(up, size=img.shape[:2], mode="bilinear", align_corners=False)[0]
    top2 = up.topk(2, dim=0).values
    margin = top2[0] - top2[1]
    assert torch.equal(up.argmax(0), labels), "recomputed labels differ from the reference's"
    res = {"input_sum": int(img.astype("int64").sum()), "net_size": net,
           "labels": ug.bands(labels.to(torch.uint8)), "rgb": ug.bands(torch.from_numpy(np.ascontiguousarray(rgb))),
           "margin": ug.bands(margin.half())}
    for i, f in enumerate(got["features"] + [got["logits"]]):
        _, c, h, w = f.shape
        res[f"stage{i}"] = ug.sample_stage(f, ug.stage_positions(h, w, c))
        res[f"stage{i}.shape"] = (c, h, w)
    counts = np.bincount(labels.numpy().ravel(), minlength=150)
    print(f"{size}: net {net}, logits {tuple(got['logits'].shape)} rms {got['logits'].pow(2).mean().sqrt():.3f}; "
          f"features rms {[round(float(f.pow(2).mean().sqrt()), 3) for f in got['features']]}; "
          f"{(counts > 0).sum()} labels used, largest share {counts.max() / counts.sum():.3f}; "
          f"margin median {margin.median():.3f}, < 0.05 at {(margin < 0.05).float().mean():.4f}")
    return res


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, infer, show, get_palette = reference_segmentor()
    g = {"seed": ug.SEED, "keys": [(k, tuple(v.shape)) for k, v in model.state_dict().items()],
         "palette": torch.tensor(get_palette("ade"), dtype=torch.uint8),
         "torch": torch.__version__, "cv2": cv2.__version__, "numpy": np.__version__}
    with torch.no_grad():
        for size in ug.SIZES:
            for key, val in run(model, infer, show, get_palette("ade"), size).items():
                g[f"{size}.{key}"] = val
    path = os.path.join(ROOT, "tests", "golden", "uniformer_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
